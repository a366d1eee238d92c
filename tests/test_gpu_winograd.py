"""int8 Winograd convolution F(2/4/6, 3) through the C ABI (-m gpu), every output element bit for bit against O.wino_conv_int8.

Every case reads back through mnnb200_conv_int8_wino_plan the launch resize planned and asserts the cell it was written for.  The
cell matrix derives its shapes from the SM count: the fused F(2,3) kernel with more than two items per CTA (consecutive items
change both their M tile and their 8-channel chunk) and with five K blocks; the batched position GEMM of F(4,3) / F(6,3) with one
item per CTA and its weights resident or streamed, with several items per CTA over two output-channel chunks (a ragged last one),
and with a K-block ring that wraps inside every item (num_kb = stages + 1, the last block 16 bytes).  Every cell has a ragged last
128-tile block, tiles that span two images, oc % 16 != 0 and ic % 16 != 0 with a non-zero input zero point, so the padded channels
of the transformed input are non-zero and only the zero weight columns cancel them.  Every cell also runs as three kernels
(execute_phases 1, 2, 4), which must equal the one-call run.

x sits 64 bytes into a buffer of random bytes (its NHWC16 channel padding zero, as the ABI requires), y 64 bytes into a poisoned
buffer: the guard bytes must come back untouched and y's channel padding zero.  Then geometry (pads, asymmetric pads, odd and
one-pixel-wide images, explicit output sizes), quantisation extremes, one execution resized many times, refusals that must leave
the previous plan working, and a captured CUDA graph replayed with a second input."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from tests.cases import random_wino_case

COMPUTE_SIZE_ERROR, NO_EXECUTION, INVALID_VALUE = 3, 4, 5
PLAN_FIELDS = ("unit", "T", "m_tiles", "Cp", "OCp", "bn", "n_chunks", "items", "grid", "one_tile", "resident_b", "stages", "num_kb")
OFF = 64                 # bytes from a buffer's start to its tensor, and from the tensor's end to the buffer's end
POISON = -77
UNITS = (2, 4, 6)
# F(4,3) / F(6,3) cells: square images whose natural output (pad 1) is 5 x 5 Winograd tiles -- 25 tiles per image, so 128-tile
# blocks straddle images
HW25 = {4: 18, 6: 28}


def lib():
    from mnn_b200 import _capi
    return _capi.lib()


def err():
    return lib().mnnb200_last_error()


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def up16(v):
    return (v + 15) // 16 * 16


def make_case(seed, unit, n, ic, oc, ih, iw, pad=(1, 1), relu=False, z_in=None):
    """random_wino_case's calibrated scales (from a small image), x of the full size, a non-zero input zero point"""
    rng = np.random.default_rng(seed)
    c = random_wino_case(rng, unit, 1, ic, oc, min(ih, 12), min(iw, 12), 1, relu)
    c["x"] = rng.integers(-128, 128, (n, ic, ih, iw)).astype(np.int8)
    c["pad"] = tuple(pad)
    c["z_in"] = z_in if z_in is not None else (c["z_in"] or 3)
    c["clamp"] = (-127, 127)
    return c


def oracle(c, unit, x=None):
    return O.wino_conv_int8(c["x"] if x is None else x, c["w"], c["ws"], c["bias"], c["in_scales"], c["in_zeros"], c["w_scales"],
                            unit, c["pad"], c["s_in"], c["z_in"], c["s_out"], c["z_out"], c["clamp"][0], c["clamp"][1], c["relu"])


def natural(c):
    _, _, ih, iw = c["x"].shape
    return ih + 2 * c["pad"][0] - 2, iw + 2 * c["pad"][1] - 2


def oracle_out(c, unit, out):
    """the oracle at an explicit output size: x extended at the bottom / right by rows and columns of z_in, which dequantise to
    +0.0f exactly like the kernels' zero fill of taps outside the image (test_zero_point_taps_equal_padding)"""
    (oh0, ow0), (oh, ow) = natural(c), out
    x = np.pad(c["x"], ((0, 0), (0, 0), (0, oh - oh0), (0, ow - ow0)), constant_values=c["z_in"])
    return oracle(c, unit, x)


def assert_same(y, ref, what):
    assert y.shape == ref.shape, (what, y.shape, ref.shape)
    diff = y != ref
    if diff.any():
        i = tuple(np.argwhere(diff)[0])
        raise AssertionError(f"{what}: {int(diff.sum())} of {diff.size} outputs differ; first at (n, c, h, w) {i}: "
                             f"{int(y[i])} != oracle {int(ref[i])}")


class Wino:
    """one int8 Winograd execution through the C ABI"""

    def __init__(self, backend, c, unit):
        from mnn_b200._capi import ConvDesc
        from mnn_b200.backend import encode_winograd_attr
        self.backend, self.unit = backend, unit
        oc, ic = c["w"].shape[:2]
        a2 = (unit + 2) ** 2
        attr = encode_winograd_attr([(0, 0, 3, 3, unit, unit, np.broadcast_to(np.asarray(c["in_scales"], np.float32), (a2,)),
                                      np.broadcast_to(np.asarray(c["in_zeros"], np.int32), (a2,)),
                                      np.broadcast_to(np.asarray(c["w_scales"], np.float32), (a2, oc)))])
        w, ws, b = (np.ascontiguousarray(c[k], t) for k, t in (("w", np.int8), ("ws", np.float32), ("bias", np.float32)))
        d = ConvDesc(ic, oc, 3, 3, 1, 1, c["pad"][0], c["pad"][1], 1, 1, 1, int(bool(c["relu"])))
        self.h = C.c_void_p()
        p = [a.ctypes.data_as(C.c_void_p) for a in (w, ws, b, attr)]
        assert lib().mnnb200_conv_int8_wino_create(backend.runtime._h, C.byref(d), *p, int(attr.size), C.byref(self.h)) == 0, err()
        self.oc, self.ic = oc, ic

    def __del__(self):
        try:
            lib().mnnb200_exec_destroy(self.h)
        except Exception:
            pass

    def resize_raw(self, n, ih, iw, s_in, z_in, s_out, z_out, cmin, cmax, out=(0, 0)):
        oh, ow = C.c_int(out[0]), C.c_int(out[1])
        st = lib().mnnb200_conv_int8_wino_resize(self.h, n, ih, iw, C.c_float(s_in), z_in, C.c_float(s_out), z_out, cmin, cmax,
                                                 C.byref(oh), C.byref(ow))
        return st, (oh.value, ow.value)

    def resize(self, c, out=None):
        """set_pad(c's pads), then resize to c's input and quantisation; the output size"""
        assert lib().mnnb200_conv_int8_set_pad(self.h, *c["pad"]) == 0, err()
        n, _, ih, iw = c["x"].shape
        st, hw = self.resize_raw(n, ih, iw, c["s_in"], c["z_in"], c["s_out"], c["z_out"], *c["clamp"], out=out or (0, 0))
        assert st == 0, err()
        self.out = hw
        return hw

    def plan(self):
        f = (C.c_int * len(PLAN_FIELDS))()
        assert lib().mnnb200_conv_int8_wino_plan(self.h, f, len(f)) == 0, err()
        return dict(zip(PLAN_FIELDS, f))

    def run(self, x, phases=(7,)):
        """x [n][ic][ih][iw] int8 through the resized execution, one execute_phases call per entry of phases; y [n][oc][oh][ow]
        after checking y's guard bytes and channel padding"""
        import torch
        n, ic, ih, iw = x.shape
        (oh, ow), cp, ocp = self.out, up16(ic), up16(self.oc)
        xh = np.zeros((n, ih, iw, cp), np.int8)
        xh[..., :ic] = x.transpose(0, 2, 3, 1)
        nx, ny = xh.size, n * oh * ow * ocp
        xb = torch.from_numpy(np.random.default_rng(nx).integers(-128, 128, nx + 2 * OFF).astype(np.int8)).cuda()
        xb[OFF:OFF + nx] = torch.from_numpy(xh.reshape(-1)).cuda()
        yb = torch.full((ny + 2 * OFF,), POISON, dtype=torch.int8, device="cuda")
        for ph in phases:
            st = lib().mnnb200_conv_int8_wino_execute_phases(self.h, C.c_void_p(xb.data_ptr() + OFF), C.c_void_p(yb.data_ptr() + OFF),
                                                             ph)
            assert st == 0, err()
        self.backend.onSync()
        yh = yb.cpu().numpy()
        guard = np.concatenate([yh[:OFF], yh[OFF + ny:]])
        assert (guard == POISON).all(), f"{int((guard != POISON).sum())} guard bytes around y were written"
        y = yh[OFF:OFF + ny].reshape(n, oh, ow, ocp)
        assert (y[..., self.oc:] == 0).all(), "NHWC16 channel padding of y must be zero"
        return np.ascontiguousarray(y[..., :self.oc].transpose(0, 3, 1, 2))


def check(ex, c, unit, what, out=None):
    """resize ex to c (explicit output size `out`), run it, compare with the oracle; (y, plan)"""
    hw = ex.resize(c, out)
    ref = oracle_out(c, unit, hw) if out else oracle(c, unit)
    y = ex.run(c["x"])
    assert_same(y, ref, what)
    return y, ex.plan()


def spans_images(n, per_image):
    """some 128-tile block of the position GEMMs holds tiles of two images"""
    return any((j * per_image) % 128 for j in range(1, n))


# ---- the cell matrix ----------------------------------------------------------------------------------------------------
CELLS = [(2, "many_items"), (2, "deep_k")] + [(u, k) for u in (4, 6)
                                              for k in ("one_tile_resident", "one_tile_streamed", "two_chunks", "ring_wrap")]


def cell_case(backend, unit, kind, sm):
    """(case, what the plan must show) for a cell, sized from the SM count"""
    a2 = (unit + 2) ** 2
    seed = unit * 100 + len(kind)
    if kind == "many_items":          # >= 2.3 items per CTA; 31 x 31 tiles per image
        ic, oc, hw = 21, 70, 62
        n = next(n for n in range(2, 1000) if -(-n * 961 // 128) * (up16(oc) // 8) >= 2.3 * sm)
        return make_case(seed, 2, n, ic, oc, hw, hw), lambda p: p["items"] >= 2.3 * sm and p["grid"] % p["n_chunks"] != 0
    if kind == "deep_k":              # Cp 608: 5 K blocks, the last 3 k-steps; >= 2 items per CTA; odd output size
        ic, oc = 601, 30
        h = next(h for h in range(9, 1001, 2) if -(-2 * ((h + 1) // 2) ** 2 // 128) * (up16(oc) // 8) >= 2 * sm)
        return make_case(seed, 2, 2, ic, oc, h, h), lambda p: p["items"] >= 2 * sm and p["num_kb"] == 5 and p["Cp"] == 608
    hw = HW25[unit]

    def images(m_tiles):              # the most 25-tile images that still need exactly m_tiles 128-tile blocks
        return (m_tiles * 128 - 1) // 25
    if kind == "one_tile_resident":
        mt = max(1, min(3, sm // a2))
        return make_case(seed, unit, images(mt), 40, 44, hw, hw), \
            lambda p: p["one_tile"] == 1 and p["resident_b"] == 1 and p["n_chunks"] == 1 and p["m_tiles"] == mt
    if kind == "one_tile_streamed":   # bn 160 x 4 K blocks = 80 KB of weights: more than stay resident
        mt = max(1, min(2, sm // a2))
        return make_case(seed, unit, images(mt), 500, 150, hw, hw), \
            lambda p: p["one_tile"] == 1 and p["resident_b"] == 0 and p["n_chunks"] == 1 and p["bn"] * 128 * p["num_kb"] > 72 * 1024
    if kind == "two_chunks":          # OC 270 -> OCp 272 in two chunks of 144: the second is ragged
        mt = -(-2 * sm // (2 * a2))
        return make_case(seed, unit, images(mt), 20, 270, hw, hw), \
            lambda p: p["n_chunks"] == 2 and p["bn"] * 2 > p["OCp"] and p["items"] >= 2 * sm and p["one_tile"] == 0
    if kind == "ring_wrap":           # num_kb = stages + 1, the last K block 16 bytes (half a k-step is TMA zero fill)
        mt = -(-2 * sm // a2)
        probe = Wino(backend, make_case(seed, unit, images(mt), 16, 13, hw, hw), unit)
        probe.resize(make_case(seed, unit, images(mt), 16, 13, hw, hw))
        stages = probe.plan()["stages"]
        return make_case(seed, unit, images(mt), stages * 128 + 11, 13, hw, hw), \
            lambda p: p["num_kb"] == stages + 1 and p["Cp"] % 128 == 16 and p["resident_b"] == 0 and p["items"] >= 2 * sm
    raise ValueError(kind)


@pytest.mark.gpu
@pytest.mark.parametrize("unit,kind", CELLS, ids=[f"F{u}-{k}" for u, k in CELLS])
def test_wino_cell_matrix(backend, unit, kind):
    sm = sm_count()
    c, reaches = cell_case(backend, unit, kind, sm)
    n, ic, _, _ = c["x"].shape
    ex = Wino(backend, c, unit)
    y, p = check(ex, c, unit, f"F({unit},3) {kind}")
    assert p["unit"] == unit and p["grid"] == min(p["items"], sm), p
    assert reaches(p), f"F({unit},3) {kind} misses its cell: {p}"
    oh, ow = natural(c)
    per_image = -(-oh // unit) * -(-ow // unit)
    assert p["T"] == n * per_image and p["T"] % 128 != 0 and spans_images(n, per_image), p
    assert c["w"].shape[0] % 16 != 0 and ic % 16 != 0 and c["z_in"] != 0
    # the same launch as three kernels: input transform, position GEMMs (EPI 2 at alpha^2 = 16 for F(2,3)), output transform
    assert_same(ex.run(c["x"], phases=(1, 2, 4)), y, f"F({unit},3) {kind} run phase by phase")


# ---- geometry -----------------------------------------------------------------------------------------------------------
def geometry_cases(unit):
    """(n, ih, iw, pad, explicit output size or None)"""
    g = [(2, 13, 9, (0, 0), None), (2, 13, 9, (2, 2), None), (2, 9, 13, (3, 3), None),    # pad 3: output rows of padding only
         (2, 13, 9, (0, 2), None), (2, 9, 13, (2, 1), None),                              # pad_h != pad_w
         (3, 1, 17, (1, 1), None), (3, 17, 1, (1, 1), None), (1, 1, 1, (1, 1), None),
         (2, 3 * unit + 1, 2 * unit + 1, (1, 1), None),                                   # OH % unit == 1
         (2, 3 * unit - 1, 2 * unit - 1, (1, 1), None)]                                   # OH % unit == unit - 1
    for pad, (dh, dw) in (((0, 0), (1, 1)), ((1, 1), (unit, unit)), ((1, 2), (1, unit)), ((0, 1), (unit, 1))):
        oh, ow = 11 + 2 * pad[0] - 2, 10 + 2 * pad[1] - 2
        g.append((2, 11, 10, pad, (oh + dh, ow + dw)))                                      # one row / one tile past the natural size
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("unit", UNITS)
def test_wino_geometry(backend, unit):
    c0 = make_case(unit + 7, unit, 1, 20, 19, 8, 8)
    ex = Wino(backend, c0, unit)
    for i, (n, ih, iw, pad, out) in enumerate(geometry_cases(unit)):
        c = dict(c0, x=np.random.default_rng(i).integers(-128, 128, (n, 20, ih, iw)).astype(np.int8), pad=pad)
        y, p = check(ex, c, unit, f"F({unit},3) n={n} {ih}x{iw} pad={pad} out={out}", out)
        assert y.shape[2:] == (out or natural(c))


def test_zero_point_taps_equal_padding():
    """taps holding z_in dequantise to +0.0f, bit-identical to the zero of a padded tap: the oracle on x framed by z_in at pad 0
    equals the oracle on x at the frame's pad, so an explicit output size can be checked on x extended by z_in"""
    for unit in UNITS:
        c = make_case(unit, unit, 2, 5, 7, 9, 7, z_in=-3)
        for ph, pw in ((1, 1), (2, 0), (1, 3)):
            framed = np.pad(c["x"], ((0, 0), (0, 0), (ph, ph), (pw, pw)), constant_values=c["z_in"])
            a = oracle(dict(c, pad=(ph, pw)), unit)
            b = oracle(dict(c, pad=(0, 0)), unit, framed)
            assert np.array_equal(a, b), (unit, ph, pw)


# ---- quantisation extremes ----------------------------------------------------------------------------------------------
def position_clamp_fraction(c, unit):
    """share of image 0's transformed input values (float64) that quantise outside [-127, 127]"""
    bt = O.wino_matrices(unit)[0].astype(np.float64)
    a = unit + 2
    (ph, pw), (oh, ow) = c["pad"], natural(c)
    x = (c["x"][0].astype(np.float64) - c["z_in"]) * c["s_in"]
    ic, ih, iw = x.shape
    hu, wu = -(-oh // unit), -(-ow // unit)
    xp = np.zeros((ic, hu * unit + 2, wu * unit + 2))
    xp[:, ph:ph + ih, pw:pw + iw] = x
    t = np.stack([xp[:, i * unit:i * unit + a, j * unit:j * unit + a] for i in range(hu) for j in range(wu)])
    v = np.einsum("ij,tcjk,lk->tcil", bt, t, bt).reshape(len(t), ic, a * a)
    q = v / np.asarray(c["in_scales"], np.float64) + np.asarray(c["in_zeros"], np.float64)
    return float(np.mean(np.abs(q) > 127.5))


@pytest.mark.gpu
@pytest.mark.parametrize("unit", UNITS)
def test_wino_quantisation_extremes(backend, unit):
    base = make_case(unit + 11, unit, 2, 20, 19, 11, 13)
    ex = Wino(backend, base, unit)
    for z in (-128, 127):
        check(ex, dict(base, z_in=z), unit, f"F({unit},3) z_in {z}")
    c = dict(base, in_scales=np.asarray(base["in_scales"], np.float32) / 8)     # the position values clamp at +-127
    assert position_clamp_fraction(c, unit) >= 0.2
    exs = Wino(backend, c, unit)      # the input scales are part of the weights' attr: a new execution
    check(exs, c, unit, f"F({unit},3) input scales / 8")
    c = dict(base, s_out=base["s_out"] / 8)
    y, _ = check(ex, c, unit, f"F({unit},3) s_out / 8")
    assert np.mean(np.abs(y.astype(int)) == 127) >= 0.05
    c = dict(base, relu=True, z_out=5)
    exr = Wino(backend, c, unit)
    y, _ = check(exr, c, unit, f"F({unit},3) ReLU, z_out 5")
    assert np.mean(y == 5) >= 0.05 and y.min() == 5
    c = dict(base, clamp=(-100, 90), s_out=base["s_out"] / 2)
    y, _ = check(ex, c, unit, f"F({unit},3) clamp (-100, 90)")
    assert y.min() == -100 and y.max() == 90


# ---- one execution, many resizes ----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("unit", UNITS)
def test_wino_many_resizes(backend, unit):
    sm = sm_count()
    first, _ = cell_case(backend, unit, "many_items" if unit == 2 else "two_chunks", sm)
    n, ic, ih, iw = first["x"].shape
    rng = np.random.default_rng(unit)
    one = dict(first, x=rng.integers(-128, 128, (1, ic, 7, 9)).astype(np.int8), s_out=first["s_out"] * 1.5,
               z_out=first["z_out"] + 3, clamp=(-120, 110))
    larger = dict(first, x=rng.integers(-128, 128, (n * 3 // 2 + 2, ic, ih, iw)).astype(np.int8), pad=(0, 2))
    ex = Wino(backend, first, unit)
    ys = []
    for c, what in ((first, "many items"), (one, "one item per CTA"), (larger, "pad (0, 2), larger: the scratch grows"),
                    (dict(first, pad=(1, 1)), "pad (1, 1), the first shape again")):
        y, p = check(ex, c, unit, f"F({unit},3) {what}")
        fresh = Wino(backend, c, unit)
        fresh.resize(c)
        assert p == fresh.plan(), (what, p, fresh.plan())
        ys.append((y, p))
    assert ys[1][1]["one_tile"] == 1 or ys[1][1]["items"] > sm
    assert ys[2][1]["T"] > ys[0][1]["T"]
    assert np.array_equal(ys[3][0], ys[0][0]) and ys[3][1] == ys[0][1]


# ---- refusals -----------------------------------------------------------------------------------------------------------
def limit_batch(unit):
    """the smallest batch of 1 x 1 images (one Winograd tile each at pad 1) whose Mpad * alpha^2 exceeds INT32_MAX"""
    a2 = (unit + 2) ** 2
    mpad_max = (0x7fffffff // a2) // 128 * 128
    return mpad_max + 1


@pytest.mark.gpu
@pytest.mark.parametrize("unit", UNITS)
def test_wino_refusals_keep_the_plan(backend, unit):
    import torch
    c = make_case(unit + 13, unit, 2, 20, 19, 11, 13)
    ex = Wino(backend, c, unit)
    f = (C.c_int * len(PLAN_FIELDS))()
    assert lib().mnnb200_conv_int8_wino_plan(ex.h, f, len(f)) == NO_EXECUTION
    assert lib().mnnb200_conv_int8_wino_execute(ex.h, None, None) == NO_EXECUTION
    y0, p0 = check(ex, c, unit, f"F({unit},3) before the refusals")
    n = limit_batch(unit)
    refusals = [("n = 0", (0, 11, 13, c["s_in"], c["z_in"], c["s_out"], c["z_out"], -127, 127), COMPUTE_SIZE_ERROR),
                ("out_scale = 0", (2, 11, 13, c["s_in"], c["z_in"], 0.0, c["z_out"], -127, 127), INVALID_VALUE),
                ("one past the Mpad * alpha^2 limit", (n, 1, 1, c["s_in"], c["z_in"], c["s_out"], c["z_out"], -127, 127),
                 COMPUTE_SIZE_ERROR)]
    for what, args, want in refusals:
        free0 = torch.cuda.mem_get_info()[0]
        st, _ = ex.resize_raw(*args)
        assert st == want, (what, st, err())
        assert torch.cuda.mem_get_info()[0] > free0 - (8 << 30), f"{what}: the refused resize allocated device memory"
        assert ex.plan() == p0, what            # before anything launches on the plan
        assert_same(ex.run(c["x"]), y0, f"F({unit},3) after the refusal {what}")
    # misaligned tensors: refused before anything launches
    xb = torch.zeros(4096, dtype=torch.int8, device="cuda")
    yb = torch.zeros(4096, dtype=torch.int8, device="cuda")
    base_x, base_y = xb.data_ptr(), yb.data_ptr()
    for dx, dy in ((1, 0), (2, 0), (0, 1), (0, 2)):
        for call in (lambda x, y: lib().mnnb200_conv_int8_wino_execute(ex.h, x, y),
                     lambda x, y: lib().mnnb200_conv_int8_wino_execute_phases(ex.h, x, y, 1)):
            assert call(C.c_void_p(base_x + dx), C.c_void_p(base_y + dy)) == INVALID_VALUE, (dx, dy)
    # plan query arguments
    assert lib().mnnb200_conv_int8_wino_plan(None, f, len(f)) == INVALID_VALUE
    assert lib().mnnb200_conv_int8_wino_plan(ex.h, None, len(f)) == INVALID_VALUE
    other = C.c_void_p()
    scale = np.ones(4, np.float32)
    assert lib().mnnb200_scale_f32_create(backend.runtime._h, 4, scale.ctypes.data_as(C.c_void_p), None, C.byref(other)) == 0
    try:
        assert lib().mnnb200_conv_int8_wino_plan(other, f, len(f)) == INVALID_VALUE
    finally:
        lib().mnnb200_exec_destroy(other)
    g = (C.c_int * 3)(-1, -1, -1)
    assert lib().mnnb200_conv_int8_wino_plan(ex.h, g, 2) == 0 and list(g) == [unit, p0["T"], -1]


# ---- graph replay -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_wino_graph_replay(backend):
    """tests/golden/wino_modern_conv.mnn (written by the reference's FlatBuffers code) through WholeNetSession, captured once
    and replayed: the recorded input must give the reference's recorded output, a second input the oracle's result"""
    import os
    from mnn_b200 import mnn_file
    from mnn_b200.session import WholeNetSession
    root = os.path.dirname(__file__)
    g = np.load(os.path.join(root, "golden", "wino_modern_conv.npz"))
    net = mnn_file.load(os.path.join(root, "golden", "wino_modern_conv.mnn"))
    conv = next(o for o in net.ops if o.conv is not None).conv
    s_in, z_in = np.float32(g["s_in"]), int(g["z_in"])
    sess = WholeNetSession(os.path.join(root, "golden", "wino_modern_conv.mnn"), 2, input_hw=(11, 13))
    assert [type(s[1]).__name__ for s in sess.steps] == ["FloatToInt8Execution", "ConvInt8WinogradExecution", "Int8ToFloatExecution"]
    last = list(sess.checkpoints)[-1]
    x2 = np.random.default_rng(3).integers(-128, 128, g["x"].shape).astype(np.int8)
    ref2 = O.wino_conv_int8(x2, conv.weight, conv.alpha, conv.bias, np.float32(g["in_scale"]), 0, np.float32(g["w_scale"]), 2, 1,
                            float(g["s_in"]), z_in, float(g["s_out"]), int(g["z_out"]), -127, 127, True)
    assert not np.array_equal(ref2, g["y"])
    sess.set_input((g["x"].astype(np.float32) - np.float32(z_in)) * s_in)
    sess.capture()
    for x, ref, what in ((g["x"], g["y"], "recorded input"), (x2, ref2, "second input"), (g["x"], g["y"], "recorded input again")):
        sess.set_input((x.astype(np.float32) - np.float32(z_in)) * s_in)
        sess.run()
        got = sess.read_int8(last)
        assert_same(got, ref.reshape(got.shape), f"graph replay, {what}")
