"""The conv-group kernel (conv_group_wgmma.cu) cell by cell (-m gpu): every tile width x K-chunk mode, the weight-tile cache and
the resident weight set under real reuse, the epilogue's arithmetic edges, the group's size limit and rebinding, and the
resnet_direct benchmark set at batch 64.  Every int8 output equals the C oracle (oracle/mnn_oracle.c) bit for bit; outputs are
poisoned before every run and NHWC16 channel padding must come back zero.

Each case reads the layer resize planned (mnnb200_conv_int8_group_plan) and asserts the cell it claims: tile width, K-chunk mode,
a ragged last n chunk, the weight-cache regime and, for the reuse cases, that the round-robin schedule really hands some CTA
several items of the layer."""
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle import oracle as O
from tests.cases import random_modern_case

pytestmark = pytest.mark.gpu

PLAN_FIELDS = ("mode", "cb", "bn", "n_chunks", "m_tiles", "num_kb", "K", "R", "TWp", "BH")
RESIDENT_BYTES = 36 * 1024
_pool = None


def pool():
    """The oracle is a plain C loop (~0.5 GMAC/s per core); ctypes drops the GIL, so references are split over threads."""
    global _pool
    if _pool is None:
        O.lib()
        _pool = ThreadPoolExecutor(max_workers=max(2, os.cpu_count() or 2))
    return _pool


class Pending:
    def __init__(self, futures):
        self.futures = futures

    def result(self):
        return np.concatenate([f.result() for f in self.futures], axis=0)


class Layer:
    """One int8 conv execution, resized, with its input uploaded and its output acquired."""

    def __init__(self, backend, c, legacy=False):
        from mnn_b200.backend import Op
        self.backend, self.c, self.legacy = backend, c, legacy
        ic, oc, kh, kw = c["w"].shape[1], c["w"].shape[0], c["w"].shape[2], c["w"].shape[3]
        self.oc = oc
        op = Op(type="ConvInt8", conv=dict(ic=ic, oc=oc, kernel=(kh, kw), stride=tuple(c["stride"]), pad=tuple(c["pad"]),
                                          dilate=tuple(c["dilate"]), group=1, relu=bool(c["relu"])),
                weight=c["w"], wscale=c["ws"], bias=c["bias"], legacy=legacy)
        self.op = op
        self.ex = None
        self.resize()

    def resize(self):
        """(Re)allocate x / y for the case's current input and quant attrs and resize the execution to them."""
        from mnn_b200.backend import QuantAttr, Tensor
        c, be = self.c, self.backend
        n, ic, ih, iw = c["x"].shape
        if self.legacy:
            qi, qo = QuantAttr(0, 0, -127, 127), QuantAttr(0, 0, -127, 127)
        else:
            qi, qo = QuantAttr(c["s_in"], c["z_in"], -128, 127), QuantAttr(c["s_out"], c["z_out"], -127, 127)
        self.xin = be.onAcquire(Tensor((n, ic, ih, iw), "int8", qi))
        be.onCopyBuffer(c["x"], self.xin)
        self.yout = Tensor((n, self.oc, 1, 1), "int8", qo)
        if self.ex is None:
            self.ex = be.onCreate([self.xin], [self.yout], self.op)
        assert self.ex.onResize([self.xin], [self.yout]) == 0
        be.onAcquire(self.yout)

    def plan(self):
        from mnn_b200 import _capi
        f = (C.c_int * len(PLAN_FIELDS))()
        assert _capi.lib().mnnb200_conv_int8_group_plan(self.ex._h, f, len(PLAN_FIELDS)) == 0
        return dict(zip(PLAN_FIELDS, f))

    def poison(self):
        self.yout.data.fill_(77)

    def output(self):
        raw = self.yout.data.cpu().numpy()
        assert (raw[..., self.oc:] == 0).all(), "NHWC16 channel padding must stay zero"
        return self.backend.onCopyBuffer(self.yout, "same")

    def reference(self, images=None):
        return self.submit(images).result()

    def submit(self, images=None):
        """Starts the oracle for all images (or the listed ones) on the thread pool, a few images per task; the result()
        of the returned object joins them."""
        c = self.c
        if self.legacy:
            bf, sx = O.fold_legacy(c["w"], c["ws"], c["bias"])
            z_in, min_v = 0, 0 if c["relu"] else -127
        else:
            bf, sx = O.fold_modern(c["w"], c["ws"], c["bias"], c["s_in"], c["z_in"], c["s_out"], c["z_out"])
            z_in, min_v = c["z_in"], c["z_out"] if c["relu"] else -127
        x = c["x"] if images is None else c["x"][list(images)]
        parts = np.array_split(np.arange(x.shape[0]), min(x.shape[0], 4 * (os.cpu_count() or 1)))
        run = lambda idx: O.conv_int8(x[idx], c["w"], c["ws"], sx, bf, stride=c["stride"], pad=c["pad"], dilate=c["dilate"],
                                      z_in=z_in, min_v=min_v, max_v=127)
        return Pending([pool().submit(run, p) for p in parts if p.size])

    def check(self, ref=None):
        y = self.output()
        ref = self.reference() if ref is None else ref
        assert y.shape == ref.shape
        assert np.array_equal(y, ref), (self.c["w"].shape, self.plan(), int(np.count_nonzero(y != ref)))
        return y


def case(rng, ic, oc, k=(1, 1), n=1, hw=(8, 8), stride=(1, 1), pad=(0, 0), dilate=(1, 1), relu=0, z_in=None):
    c = random_modern_case(rng, ic, oc, k[0], k[1], n, hw[0], hw[1], stride, pad, relu, dilate)
    if z_in is not None:
        c["z_in"] = z_in
    return c


def run_group(backend, layers):
    from mnn_b200.backend import ConvGroupExecution
    for L in layers:
        assert ConvGroupExecution.groupable(L.ex), L.plan()
    grp = ConvGroupExecution(backend, [L.ex for L in layers])
    assert grp.bind([L.xin for L in layers], [L.yout for L in layers]) == 0
    for L in layers:
        L.poison()
    assert grp.onExecute() == 0
    backend.onSync()
    return grp


# ---- what a plan says about the kernel's paths (restated from conv_group_wgmma.cu) ------------------------------------
def form(p):
    return "1x1" if p["mode"] == 0 else f"cb{p['cb']}"


def regime(p):
    """The producer's weight-tile path (conv_group_wgmma.cu, the TMA producer): `untagged` (num_kb > 256 on an implicit-GEMM
    layer), `resident` (the `resident` condition of the cb >= 64 branch), else the 4 tagged slots."""
    if p["mode"] == 1 and p["num_kb"] > 256:
        return "untagged"
    if p["mode"] == 1 and p["cb"] >= 64 and p["num_kb"] > 4 and p["bn"] * p["cb"] % 1024 == 0 \
            and p["num_kb"] * p["bn"] * p["cb"] <= RESIDENT_BYTES:
        return "resident"
    return "slots"


def ragged_n(L, p):
    ocp = (L.oc + 15) // 16 * 16
    return ocp - (p["n_chunks"] - 1) * p["bn"] < p["bn"]


def ragged_m(L, p):
    """The last M tile is part empty: 128-row tiles over M (mode 0), or R row boxes per tile over the layer's row boxes."""
    n = L.c["x"].shape[0]
    oh, ow = L.yout.shape[2], L.yout.shape[3]
    if p["mode"] == 0:
        return (n * oh * ow) % 128 != 0
    rowboxes = n * (oh // p["BH"]) * (-(-ow // 128))
    return rowboxes % p["R"] != 0


def schedule(layers, sm_count):
    """group_build's schedule: items (layer, n chunk) in member order, M tile outer, n chunk inner; item i -> CTA i mod grid."""
    items = [(l, nc) for l, L in enumerate(layers) for p in [L.plan()] for _ in range(p["m_tiles"]) for nc in range(p["n_chunks"])]
    grid = min(len(items), sm_count)
    return [items[c::grid] for c in range(grid)]


def reuse(ctas, l):
    """(most items of layer l on one CTA, most distinct n chunks of layer l on one CTA)"""
    return (max(sum(1 for it in row if it[0] == l) for row in ctas),
            max(len({it[1] for it in row if it[0] == l}) for row in ctas))


def acc_u(c, z_in=None):
    """int64 sum over the taps of (x + 128) * w, padded taps holding z_in: the accumulator the epilogue requantises."""
    x, w = c["x"].astype(np.int64) + 128, c["w"].astype(np.int64)
    (sh, sw), (ph, pw), (dh, dw) = c["stride"], c["pad"], c["dilate"]
    z = c["z_in"] if z_in is None else z_in
    n, ic, ih, iw = x.shape
    oc, _, kh, kw = w.shape
    oh, ow = O.conv_out_size(ih, kh, sh, ph, dh), O.conv_out_size(iw, kw, sw, pw, dw)
    xp = np.full((n, ic, ih + 2 * ph + sh * oh, iw + 2 * pw + sw * ow), z + 128, np.int64)
    xp[:, :, ph:ph + ih, pw:pw + iw] = x
    acc = np.zeros((n, oc, oh, ow), np.int64)
    for a in range(kh):
        for b in range(kw):
            win = xp[:, :, a * dh:a * dh + sh * oh:sh, b * dw:b * dw + sw * ow:sw]
            acc += np.einsum("nchw,oc->nohw", win, w[:, :, a, b])
    return acc


# ---- 0. the plan query -------------------------------------------------------------------------------------------------
def test_group_plan_query_status(backend):
    from mnn_b200 import _capi
    from mnn_b200.backend import Op, QuantAttr, Tensor
    rng = np.random.default_rng(1)
    c = case(rng, 16, 16, (3, 3), 1, (9, 9), (1, 3), (1, 1))
    op = Op(type="ConvInt8", conv=dict(ic=16, oc=16, kernel=(3, 3), stride=(1, 3), pad=(1, 1), dilate=(1, 1), group=1, relu=False),
            weight=c["w"], wscale=c["ws"], bias=c["bias"])
    xin = backend.onAcquire(Tensor((1, 16, 9, 9), "int8", QuantAttr(c["s_in"], c["z_in"], -128, 127)))
    yout = Tensor((1, 16, 1, 1), "int8", QuantAttr(c["s_out"], c["z_out"], -127, 127))
    ex = backend.onCreate([xin], [yout], op)
    f = (C.c_int * len(PLAN_FIELDS))(*([-7] * len(PLAN_FIELDS)))
    assert _capi.lib().mnnb200_conv_int8_group_plan(ex._h, f, len(PLAN_FIELDS)) == 4      # NO_EXECUTION before resize
    assert ex.onResize([xin], [yout]) == 0
    assert _capi.lib().mnnb200_conv_int8_group_plan(ex._h, f, len(PLAN_FIELDS)) == 2      # stride_w 3: not on the group kernel
    assert list(f) == [-7] * len(PLAN_FIELDS)
    L = Layer(backend, case(rng, 40, 100, (3, 3), 2, (12, 20), pad=(1, 1), z_in=2))
    p = L.plan()
    assert (p["mode"], p["cb"], p["bn"], p["n_chunks"], p["K"], p["TWp"]) == (1, 16, 112, 1, 16 * 28, 24)
    assert p["BH"] * p["TWp"] * p["R"] <= 128 and p["m_tiles"] == -(-(2 * (12 // p["BH"])) // p["R"])


# ---- A. every tile width x K-chunk mode in one group launch ------------------------------------------------------------
BNS = (16, 32, 48, 64, 80, 96, 112, 128)
RAGGED_OCP = {80: 144, 112: 208, 128: 368}     # bn 80 / 112 / 128 with a last n chunk of 64 / 96 / 112 columns
# implicit-GEMM geometries: kernel, stride, pad, dilation, batch, input size.  All padded; BH > 1 with R = 2 in the last
MODE1_GEOM = [((3, 3), (1, 1), (1, 1), (1, 1), 1, (13, 13)), ((3, 3), (2, 2), (1, 1), (1, 1), 1, (25, 25)),
              ((3, 3), (1, 1), (2, 2), (2, 2), 2, (13, 13)), ((3, 3), (1, 1), (1, 1), (1, 1), 3, (8, 7))]
FORM_IC = {"1x1": (100, 300), "cb128": (120, 120), "cb64": (60, 60), "cb16": (21, 40)}


def matrix_cells():
    cells = []
    for f, form_name in enumerate(("1x1", "cb128", "cb64", "cb16")):
        for i, bn in enumerate(BNS):
            ocp = RAGGED_OCP.get(bn, bn)
            oc = ocp - (5 if bn in RAGGED_OCP else 3)
            ic = FORM_IC[form_name][i % 2]
            # 3x3 everywhere in mode 1: cb 128 -> 9 K blocks of bn x 128 bytes, cb 64 -> 9 of bn x 64 bytes (resident up to 36 KB)
            res = (form_name == "cb128" and bn <= 32) or (form_name == "cb64" and bn <= 64)
            cells.append(dict(form=form_name, bn=bn, oc=oc, ic=ic, ragged=bn in RAGGED_OCP, regime="resident" if res else "slots",
                              relu=(8 * f + i) % 2, geom=i % 4, z_in=(3, -4, 5, -2)[i % 4]))
    return cells


def test_conv_group_width_by_chunk_matrix(backend):
    rng = np.random.default_rng(2024)
    layers, seen = [], set()
    for cell in matrix_cells():
        if cell["form"] == "1x1":
            n, hw = ((1, (15, 19)), (2, (9, 11)))[cell["geom"] % 2]
            c = case(rng, cell["ic"], cell["oc"], (1, 1), n, hw, relu=cell["relu"], z_in=cell["z_in"])
        else:
            k, st, pad, dl, n, hw = MODE1_GEOM[cell["geom"]]
            c = case(rng, cell["ic"], cell["oc"], k, n, hw, st, pad, dl, relu=cell["relu"], z_in=cell["z_in"])
        L = Layer(backend, c)
        p = L.plan()
        assert (form(p), p["bn"]) == (cell["form"], cell["bn"]), (cell, p)
        assert ragged_n(L, p) == cell["ragged"], (cell, p)
        assert regime(p) == cell["regime"], (cell, p)
        assert p["m_tiles"] >= 2 and ragged_m(L, p), (cell, p)
        if p["mode"] == 1:
            assert min(c["pad"]) > 0 and c["z_in"] != 0
        seen.add((form(p), p["bn"]))
        layers.append(L)
    assert len(seen) == 32
    refs = [L.submit() for L in layers]
    run_group(backend, layers)
    grouped = [L.check(r.result()) for L, r in zip(layers, refs)]
    # each member alone: on a one-layer group (variant 2) and on the mma.sync kernel (variant 1, no code shared with the group)
    for L, y in zip(layers, grouped):
        for variant in (2, 1):
            L.ex.set_variant(variant)
            L.poison()
            assert L.ex.onExecute([L.xin], [L.yout]) == 0
            backend.onSync()
            assert np.array_equal(L.output(), y), (variant, L.plan())


# ---- B. weight-tile reuse: the 4 tagged slots, the resident set, untagged blocks ---------------------------------------
def test_conv_group_weight_tile_reuse(backend):
    sm = backend.runtime.sm_count
    rng = np.random.default_rng(77)

    def images(tiles_per_image, n_chunks=1):
        """images for more than 2 x SM count items of the layer"""
        m_tiles = (2 * sm) // n_chunks + 1
        return -(-m_tiles * tiles_per_image[1] // tiles_per_image[0])

    px = (135, 128)          # a 9 x 15 map: 135 pixels per image, 128 rows per M tile
    rb = (4, 1)              # a 16 x 32 output: 4 row boxes of 4 x 32 pixels per image, one per M tile
    specs = []   # (name, case, expected (form, bn, n_chunks, regime), extra plan checks)
    # 4 slots, mode 0: 2 K blocks, 5 n chunks of 112 (a CTA's next item is another n chunk: 10 keys through 4 slots)
    specs.append(("slots_5chunks", case(rng, 200, 557, (1, 1), images(px, 5), (9, 15), z_in=-3),
                  ("1x1", 112, 5, "slots"), dict(num_kb=2)))
    # 4 slots, one n chunk: every item of a CTA hits the slots its first item filled
    specs.append(("slots_hit", case(rng, 256, 30, (1, 1), images(px), (9, 15), relu=1),
                  ("1x1", 32, 1, "slots"), dict(num_kb=2)))
    for ic, kb in ((600, 5), (700, 6), (800, 7)):     # just past the 4 slots, around the 6-stage ring
        specs.append((f"slots_kb{kb}", case(rng, ic, 13, (1, 1), images(px), (9, 15), relu=kb % 2),
                      ("1x1", 16, 1, "slots"), dict(num_kb=kb)))
    # resident: 3x3 x 64 at bn 64 = 9 x 4 KB, exactly the 36 KB
    specs.append(("resident_36k", case(rng, 64, 61, (3, 3), images(rb), (16, 32), pad=(1, 1), z_in=4),
                  ("cb64", 64, 1, "resident"), dict(num_kb=9, BH=4, R=1)))
    # resident: 1x5 x 64, 5 n chunks of 112 = 5 x 7 KB: a CTA switches n chunk between items and reloads the set
    specs.append(("resident_5chunks", case(rng, 64, 557, (1, 5), images(rb, 5), (16, 32), pad=(0, 2), relu=1, z_in=-2),
                  ("cb64", 112, 5, "resident"), dict(num_kb=5)))
    # resident: 3x3 x 128 at bn 32 = 9 x 4 KB (cb 128)
    specs.append(("resident_cb128", case(rng, 128, 29, (3, 3), images(rb), (16, 32), pad=(1, 1), z_in=1),
                  ("cb128", 32, 1, "resident"), dict(num_kb=9)))
    # two resident layers of identical geometry, different weights, back to back: the set must be reloaded between them
    for t in range(2):
        specs.append((f"resident_twin{t}", case(rng, 64, 13, (3, 3), images(rb), (16, 32), pad=(1, 1), z_in=-5),
                      ("cb64", 16, 1, "resident"), dict(num_kb=9)))
    # untagged: more than 256 K blocks on a small map (cb 128: 9 taps x 32 chunks; cb 16: 121 taps x 17 chunks + 1 -> 258 blocks)
    specs.append(("untagged_cb128", case(rng, 4096, 40, (3, 3), 3, (7, 7), pad=(1, 1), z_in=2),
                  ("cb128", 48, 1, "untagged"), dict(num_kb=288)))
    specs.append(("untagged_cb16", case(rng, 272, 24, (11, 11), 1, (12, 12), pad=(5, 5), relu=1, z_in=-1),
                  ("cb16", 32, 1, "untagged"), dict(num_kb=258)))

    layers = [Layer(backend, c) for _, c, _, _ in specs]
    ctas = schedule(layers, sm)
    for l, ((name, c, (f, bn, nch, reg), extra), L) in enumerate(zip(specs, layers)):
        p = L.plan()
        assert (form(p), p["bn"], p["n_chunks"], regime(p)) == (f, bn, nch, reg), (name, p)
        assert all(p[k] == v for k, v in extra.items()), (name, p)
        if reg != "untagged":
            most, distinct = reuse(ctas, l)
            assert most >= 2, (name, most)                           # some CTA computes the layer twice or more
            assert nch == 1 or distinct >= 2, (name, distinct)       # ... with different n chunks where there are several
    t0 = [s[0] for s in specs].index("resident_twin0")
    assert layers[t0].plan() == layers[t0 + 1].plan() and not np.array_equal(specs[t0][1]["w"], specs[t0 + 1][1]["w"])
    assert all(any(it[0] == t0 for it in row) and any(it[0] == t0 + 1 for it in row) for row in ctas)   # every CTA runs both
    refs = [L.submit() for L in layers]
    run_group(backend, layers)
    wrong = {}                  # every layer is checked: which ones a wrong cache key breaks tells which key field it is
    for (name, c, _, _), L, r in zip(specs, layers, refs):
        y, ref = L.output(), r.result()
        if not np.array_equal(y, ref):
            wrong[name] = int(np.count_nonzero(y != ref))
        assert (np.abs(ref.astype(int)) == 127).mean() < 0.5, name
    assert not wrong, wrong


# ---- C. epilogue arithmetic --------------------------------------------------------------------------------------------
def extreme_case(rng, ic, oc, k, n, hw, pad=(0, 0), z_in=0):
    """x, w in {-128, 127} in sign patterns (whole pixels / rows of one sign, and random signs); wscale per channel so that the
    largest |output| is about 110: the accumulators reach their bounds without the outputs saturating."""
    c = case(rng, ic, oc, k, n, hw, pad=pad, z_in=z_in)
    x = np.where(rng.random(c["x"].shape) < 0.5, -128, 127).astype(np.int8)
    x[:, :, :4, :4] = 127          # windows of all-127 pixels (x + 128 = 255) and of all -128 (x + 128 = 0)
    x[:, :, -4:, -4:] = -128
    w = np.where(rng.random(c["w"].shape) < 0.5, -128, 127).astype(np.int8)
    w[0::4] = 127
    w[1::4] = -128
    c["x"], c["w"] = x, w
    real = acc_u(c) - (c["z_in"] + 128) * w.astype(np.int64).reshape(oc, -1).sum(1)[None, :, None, None]
    sx = np.float32(c["s_in"]) / np.float32(c["s_out"])
    c["ws"] = (110.0 / (np.abs(real).max(axis=(0, 2, 3)) * sx)).astype(np.float32)
    c["bias"] = (rng.uniform(-1, 1, oc) * 5 * c["s_out"]).astype(np.float32)
    return c


def tie_case(rng, ic, oc, k, n, hw, pad=(0, 0)):
    """legacy fold (scale_x = 1, biasFloat = b * scale) with scales 2^-1 / 2^-2: f = (sum x w + b) * scale exactly, so
    +-k.5 occurs on every path"""
    c = case(rng, ic, oc, k, n, hw, pad=pad, z_in=0)
    c["x"] = rng.integers(-3, 4, c["x"].shape).astype(np.int8)
    c["w"] = rng.integers(-3, 4, c["w"].shape).astype(np.int8)
    c["ws"] = np.where(np.arange(oc) % 2 == 0, 0.5, 0.25).astype(np.float32)
    c["bias"] = rng.integers(-20, 21, oc).astype(np.int32)
    return c


def test_conv_group_epilogue_arithmetic(backend):
    rng = np.random.default_rng(31)
    layers, kinds = [], []
    # accumulator bounds: K = 128 exactly (the small-accumulator path), just above it, and past 2^24
    for (ic, k, pad, z_in, want_K, small) in ((128, (1, 1), (0, 0), 0, 128, True), (32, (2, 2), (0, 0), 0, 128, True),
                                               (144, (1, 1), (0, 0), 3, 144, False)):
        layers.append(Layer(backend, extreme_case(rng, ic, 40, k, 2, (9, 11), pad, z_in)))
        kinds.append(("bound", want_K, small))
    layers.append(Layer(backend, extreme_case(rng, 512, 24, (3, 3), 1, (6, 6), (1, 1), -128)))
    kinds.append(("bound", 4608, False))
    # ties on both requant paths, in both layer modes
    for (ic, k, pad, small) in ((64, (1, 1), (0, 0), True), (200, (1, 1), (0, 0), False), (32, (2, 2), (1, 1), True),
                                (32, (3, 3), (1, 1), False)):
        layers.append(Layer(backend, tie_case(rng, ic, 34, k, 2, (9, 10), pad), legacy=True))
        kinds.append(("tie", None, small))
    # clamping: about 30 % of the outputs saturate at each end
    c = case(rng, 64, 48, (3, 3), 2, (10, 12), pad=(1, 1), z_in=4)
    real = acc_u(c) - (c["z_in"] + 128) * c["w"].astype(np.int64).reshape(48, -1).sum(1)[None, :, None, None]
    c["ws"] = np.full(48, 240.0 / (real.std() * np.float32(c["s_in"]) / np.float32(c["s_out"])), np.float32)
    c["bias"] = np.zeros(48, np.float32)
    layers.append(Layer(backend, c))
    kinds.append(("clamp", None, False))

    refs = [L.submit() for L in layers]
    for L, (kind, want_K, small) in zip(layers, kinds):
        p = L.plan()
        if kind == "bound":
            assert p["K"] == want_K and (p["K"] <= 128) == small, p
            a = np.abs(acc_u(L.c)).max()
            assert a >= (0.9 * 2 ** 22 if small else (2 ** 22 if want_K == 144 else 2 ** 24)), (p, a)
        elif kind == "tie":
            assert (p["K"] <= 128) == small, p
            numer = acc_u(L.c) - 128 * L.c["w"].astype(np.int64).reshape(L.oc, -1).sum(1)[None, :, None, None] \
                + L.c["bias"].astype(np.int64)[None, :, None, None]
            f = numer * L.c["ws"].astype(np.float64)[None, :, None, None]
            # ties +-k.5 with k even: rounding half away from zero and half to even disagree there
            a = np.abs(f)
            even_tie = (a % 1 == 0.5) & (np.trunc(a) % 2 == 0) & (a < 127)
            assert (even_tie & (f > 0)).sum() >= 10 and (even_tie & (f < 0)).sum() >= 10
            assert (np.abs(f) >= 127).mean() < 0.01
    run_group(backend, layers)
    for L, (kind, _, _), r in zip(layers, kinds, refs):
        y = L.check(r.result()).astype(int)
        if kind == "clamp":
            assert 0.2 <= (y == 127).mean() <= 0.4 and 0.2 <= (y == -127).mean() <= 0.4, ((y == 127).mean(), (y == -127).mean())
        else:
            assert (np.abs(y) == 127).mean() < 0.05


# ---- D. group structure ------------------------------------------------------------------------------------------------
SMALL = [  # ic, oc, k, n, (ih, iw), stride, pad
    (16, 24, (1, 1), 1, (9, 9), (1, 1), (0, 0)), (24, 40, (3, 3), 1, (8, 8), (1, 1), (1, 1)),
    (40, 16, (1, 1), 2, (5, 7), (1, 1), (0, 0)), (8, 32, (3, 3), 1, (9, 9), (2, 2), (1, 1)),
    (64, 48, (3, 3), 1, (6, 6), (1, 1), (1, 1)), (32, 20, (2, 2), 1, (7, 7), (1, 1), (0, 0)),
    (48, 130, (1, 1), 1, (8, 8), (1, 1), (0, 0)), (20, 36, (5, 5), 1, (9, 9), (1, 1), (2, 2)),
]


def small_layer(backend, rng, i, z_in=None):
    ic, oc, k, n, hw, st, pad = SMALL[i % len(SMALL)]
    return Layer(backend, case(rng, ic, oc, k, n, hw, st, pad, relu=i % 2, z_in=z_in))


def test_conv_group_64_members_and_65_refused(backend):
    from mnn_b200 import _capi
    rng = np.random.default_rng(64)
    layers = [small_layer(backend, rng, i) for i in range(64)]
    refs = [L.submit() for L in layers]
    run_group(backend, layers)
    for L, r in zip(layers, refs):
        L.check(r.result())
    arr = (C.c_void_p * 65)(*([L.ex._h.value for L in layers] + [layers[0].ex._h.value]))
    h = C.c_void_p()
    assert _capi.lib().mnnb200_conv_group_create(backend.runtime._h, arr, 65, C.byref(h)) == 2    # NOT_SUPPORT
    assert not h.value


def test_conv_group_rebind_and_reresize(backend):
    from mnn_b200.backend import ConvGroupExecution
    rng = np.random.default_rng(5)
    layers = [small_layer(backend, rng, 0, z_in=2), small_layer(backend, rng, 1, z_in=0), small_layer(backend, rng, 4, z_in=-3)]
    grp = run_group(backend, layers)
    for L in layers:
        L.check()
    # rebind the same group to freshly allocated x / y holding new inputs: the new y is right, the old y is not written
    old = [L.yout for L in layers]
    for L in layers:
        L.c["x"] = rng.integers(-128, 128, L.c["x"].shape).astype(np.int8)
        L.resize()
        L.poison()
    for y in old:
        y.data.fill_(77)
    assert grp.bind([L.xin for L in layers], [L.yout for L in layers]) == 0
    assert grp.onExecute() == 0
    backend.onSync()
    for L in layers:
        L.check()
    for y in old:
        assert (y.data.cpu().numpy() == 77).all(), "a rebound group wrote its old output"
    # re-resize the padded 3x3 member (z_in 0: no border tables) to batch 3 and z_in 6, rebind, run again
    before = layers[1].plan()
    c = layers[1].c
    c["x"] = rng.integers(-128, 128, (3,) + c["x"].shape[1:]).astype(np.int8)
    c["z_in"] = 6
    layers[1].resize()
    assert layers[1].plan()["m_tiles"] > before["m_tiles"]
    assert ConvGroupExecution.groupable(layers[1].ex)
    assert grp.bind([L.xin for L in layers], [L.yout for L in layers]) == 0
    for L in layers:
        L.poison()
    assert grp.onExecute() == 0
    backend.onSync()
    for L in layers:
        L.check()


def test_conv_group_solo_path_alternating_pairs(backend):
    """an implicit-GEMM conv alone (auto variant) runs on a one-layer group that is rebuilt when x or y change"""
    from mnn_b200.backend import Tensor
    rng = np.random.default_rng(11)
    L = Layer(backend, case(rng, 48, 80, (3, 3), 2, (11, 13), pad=(1, 1), relu=1, z_in=-4))
    assert L.plan()["mode"] == 1
    pairs = []
    for t in range(2):
        x = rng.integers(-128, 128, L.c["x"].shape).astype(np.int8)
        xin = backend.onAcquire(Tensor(L.xin.shape, "int8", L.xin.quant))
        backend.onCopyBuffer(x, xin)
        yout = backend.onAcquire(Tensor(L.yout.shape, "int8", L.yout.quant))
        L.c["x"] = x
        pairs.append((xin, yout, L.reference()))
    for rep in range(4):
        xin, yout, ref = pairs[rep % 2]
        yout.data.fill_(77)
        assert L.ex.onExecute([xin], [yout]) == 0
        backend.onSync()
        for xo, yo, r in pairs[:rep + 1]:           # this pair's output is right, the other's still holds its last result
            assert (yo.data.cpu().numpy()[..., L.oc:] == 0).all()
            assert np.array_equal(backend.onCopyBuffer(yo, "same"), r)


# ---- E. the resnet_direct benchmark set at batch 64 --------------------------------------------------------------------
def test_conv_group_resnet_direct_set_batch64(backend):
    """bench.py --workload resnet_direct's 13 layers with its generators and quant attrs, as one group: every output equals the
    per-layer mma.sync kernel (variant 1, no code shared with the group kernel); images 0, 1 and 63 (the last M tiles) equal the
    oracle.  Again with an input zero point of 3 (border correction tables on every layer)."""
    import torch
    from bench_workloads import RESNET_LAYERS
    from mnn_b200.backend import ConvGroupExecution
    B = 64
    rng = np.random.default_rng(0)
    g = torch.Generator(device="cpu").manual_seed(0)
    layers = []
    for (Cn, HW) in RESNET_LAYERS:
        w = rng.integers(-127, 128, (Cn, Cn, 3, 3)).astype(np.int8)
        ws = (rng.uniform(0.003, 0.012, Cn) / np.sqrt(Cn * 9)).astype(np.float32)
        bias = rng.uniform(-0.5, 0.5, Cn).astype(np.float32)
        x = torch.randint(-127, 128, (B, HW, HW, Cn), generator=g, dtype=torch.int8).permute(0, 3, 1, 2).contiguous().numpy()
        c = dict(x=x, w=w, ws=ws, bias=bias, s_in=0.05, s_out=0.1, z_in=0, z_out=0, stride=(1, 1), pad=(1, 1), dilate=(1, 1),
                 relu=1)
        layers.append(Layer(backend, c))
    for z_in in (0, 3):
        if z_in:
            for L in layers:
                L.c["z_in"] = z_in
                L.resize()
        refs = [L.submit((0, 1, B - 1)) for L in layers]
        grp = ConvGroupExecution(backend, [L.ex for L in layers])
        assert grp.bind([L.xin for L in layers], [L.yout for L in layers]) == 0
        for L in layers:
            L.poison()
        assert grp.onExecute() == 0
        backend.onSync()
        grouped = [L.yout.data.clone() for L in layers]
        for L, yg, r in zip(layers, grouped, refs):
            y = L.output()
            assert np.array_equal(y[[0, 1, B - 1]], r.result()), (L.c["w"].shape, z_in)
            L.ex.set_variant(1)
            L.poison()
            assert L.ex.onExecute([L.xin], [L.yout]) == 0
            backend.onSync()
            assert torch.equal(L.yout.data, yg), (L.c["w"].shape, z_in, int((L.yout.data != yg).sum()))
            L.ex.set_variant(0)
        del grp
