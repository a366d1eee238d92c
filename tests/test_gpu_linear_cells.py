"""The LLM linear layer's tensor-core GEMM in every launch cell its create paths reach (-m gpu), bit for bit against the oracles.

Each case derives its shape from the SM count, reads back through mnnb200_linear_w8_plan which launch execute makes (path, bn,
n chunks, m tiles, work items, grid, one-tile mode, resident B, ring stages, K blocks), asserts the cell it was written for, and
runs each weight form the kernel takes there: 8-bit per channel (the single-CTA GEMM forced by variant 2; auto runs >= 256
tokens on the CTA pair), 8-bit K-blocked, 4-bit per channel and 4-bit K-blocked.  The output sits in a NaN-filled buffer 3 rows
longer than tokens * oc: every output must be written and the guard rows must stay NaN.  The oracles are scalar C, so they see
only sampled rows -- rows 0, 1, 63, 64 and 127 of every 128-row m tile and every row of the last one.  For >= 2 tokens an output
row depends only on its own token (per-token abs-max quantisation), so the oracle of the sampled rows is the oracle of the layer
at those rows; every sampled row spans every n chunk, so every CTA is checked."""
import ctypes as C

import numpy as np
import pytest

from oracle import w4_oracle as W
from tests.test_gpu_dispatch import create_linear, linear_oracle

pytestmark = pytest.mark.gpu

NOT_SUPPORT, NO_EXECUTION, INVALID_VALUE = 2, 4, 5
PLAN_FIELDS = ("path", "bn", "n_chunks", "m_tiles", "items", "grid", "one_tile", "resident_b", "stages", "num_kb", "smem")
GEMV, GEMM, PAIR, REFUSED = 0, 1, 2, -1
GUARD_ROWS = 3
FORMS = ("w8", "w8_blocked", "w4", "w4_blocked")


def lib():
    from mnn_b200 import _capi
    return _capi.lib()


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def up(v, m):
    return -(-v // m) * m


def pick_bn(ocp, m_tiles, sms, max_bn):
    """capi.cu pick_bn: equal n chunks of at most max_bn columns, more of them while m_tiles * chunks would not fill the SMs"""
    chunks = -(-ocp // max_bn)
    if m_tiles * chunks < sms:
        chunks = max(chunks, min(sms // m_tiles, ocp // 32))
    return up(-(-ocp // chunks), 16)


class Layer:
    """one linear execution created through the C ABI, with its host data: form is one of FORMS, bs the block size of a
    blocked form (0 per channel)"""

    def __init__(self, backend, form, ic, oc, bs=0, seed=0):
        self.backend, self.form, self.ic, self.oc = backend, form, ic, oc
        self.bs = bs if form.endswith("blocked") else 0
        self.blocks = ic // self.bs if self.bs else 1
        assert ic % self.blocks == 0
        rng = np.random.default_rng(seed)
        w4 = form.startswith("w4")
        self.bits = 4 if w4 else 8
        self.alpha = rng.uniform(0.001, 0.01, (oc, self.blocks)).astype(np.float32)
        self.wzero = (rng.uniform(-0.01, 0.09, (oc, self.blocks)) if w4 else rng.uniform(-0.05, 0.05, (oc, self.blocks))).astype(np.float32)
        self.bias = rng.uniform(-1, 1, oc).astype(np.float32)
        self.w = W.pack_w4(rng.integers(-8, 8, (oc, ic))) if w4 else rng.integers(-128, 128, (oc, ic), dtype=np.int8)
        if form == "w8":        # the 8-bit per-channel form takes alpha / wzero [oc]
            self.alpha, self.wzero = self.alpha[:, 0].copy(), self.wzero[:, 0].copy()
        self.h = self.create()
        self.tokens = 0

    def create(self):
        """a new execution of this layer"""
        st, h = create_linear(self.backend, self.ic, self.oc, self.w, self.alpha, self.wzero, self.bias, self.bits)
        assert st == 0, lib().mnnb200_last_error()
        return h

    def destroy(self):
        lib().mnnb200_exec_destroy(self.h)

    def resize(self, tokens, variant):
        assert lib().mnnb200_linear_w8_resize(self.h, tokens) == 0, lib().mnnb200_last_error()
        assert lib().mnnb200_conv_int8_set_variant(self.h, variant) == 0
        self.tokens = tokens
        return self.plan()

    def plan(self):
        f = (C.c_int * len(PLAN_FIELDS))()
        assert lib().mnnb200_linear_w8_plan(self.h, f, len(f)) == 0, lib().mnnb200_last_error()
        return dict(zip(PLAN_FIELDS, f))

    def inputs(self, seed):
        import torch
        g = torch.Generator(device="cuda")
        g.manual_seed(seed)
        return torch.rand((self.tokens, self.ic), generator=g, device="cuda") * 2 - 1

    def execute(self, x, y_offset=0):
        """y = layer(x) in a NaN-filled buffer of tokens + GUARD_ROWS rows, y_offset floats into it; checks that every output was
        written and the guard rows were not.  Returns the output on the device."""
        import torch
        n = self.tokens * self.oc
        buf = torch.full((n + GUARD_ROWS * self.oc + y_offset,), float("nan"), dtype=torch.float32, device="cuda")
        y = buf[y_offset:y_offset + n]
        st = lib().mnnb200_linear_w8_execute(self.h, C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()))
        assert st == 0, lib().mnnb200_last_error()
        self.backend.onSync()
        unwritten = int(torch.isnan(y).sum())
        assert unwritten == 0, f"{unwritten} of {n} outputs left unwritten"
        assert bool(torch.isnan(buf[:y_offset]).all() and torch.isnan(buf[y_offset + n:]).all()), "write past the output"
        return y.view(self.tokens, self.oc)

    def oracle(self, x):
        return linear_oracle(x, self.w, self.alpha, self.wzero, self.bias, self.bits)

    def check(self, x, y, what):
        """the sampled rows of y equal the oracle's bit for bit"""
        rows = sampled_rows(self.tokens)
        ref = self.oracle(x[rows].cpu().numpy())
        got = y[rows].cpu().numpy()
        bad = got != ref
        if bad.any():
            r, c = np.argwhere(bad)[0]
            raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} sampled outputs differ; first at row {rows[r]} column "
                                 f"{c}: {got[r, c]!r} against {ref[r, c]!r}")


def sampled_rows(tokens):
    """rows {0, 1, 63, 64, 127} of every 128-row m tile and every row of the last one (at least 2 rows: one token is the other
    arithmetic)"""
    last = (tokens - 1) // 128 * 128
    rows = {r for t in range(0, last, 128) for r in (t, t + 1, t + 63, t + 64, t + 127)} | set(range(last, tokens))
    rows = sorted(rows)
    assert len(rows) >= 2
    return rows


def variant_of(form, tokens):
    """the single-CTA GEMM: auto runs 8-bit per-channel layers of >= 256 tokens on the CTA pair, so those force variant 2"""
    return 2 if form == "w8" and tokens >= 256 else 0


def barely_persistent(sms, max_bn):
    """(tokens, oc): m_tiles * n_chunks between sms + 1 and sms + 8 at chunks of max_bn columns, the chunk count not dividing sms
    (a CTA's second item lies in another n chunk), a ragged last m tile"""
    for c in range(3, 64):
        m = sms // c + 1
        if sms % c and m * c - sms <= 8:
            return (m - 1) * 128 + 77, c * max_bn - 16
    raise AssertionError(f"no barely persistent shape for {sms} SMs")


# cell -> (shape(sms, form) -> (tokens, ic, oc, bs; bs is ignored per channel), check(plan, sms, tokens, form): the plan fields
# that put the form in the cell)
def _many_chunks(sms, form):
    return 4096, 2048, 6144, 64 if form == "w8_blocked" else 128


def _barely(sms, form):
    tokens, oc = barely_persistent(sms, 128 if form.endswith("blocked") else 256)
    return tokens, 2048, oc, 64


def _resident(sms, form):
    return sms * 128 + 40, 256, 40, 32


def _streamed(sms, form):
    return sms * 128 + 40, 2048, 120 if form.endswith("blocked") else 200, 64


def _ring_wraps(sms, form):
    return 700, 5632, 2000, 512


def _partial_k(sms, form):
    return 2000, 936 if form == "w8" else 1056, 777, 32


def _odd_oc(sms, form):
    return 333, 1000 if form in ("w8", "w4") else 1024, 1001, 32


def _bn16(sms, form):
    return 300, 512, 9, 32


def _check_many(pl, sms, tokens, form):
    assert pl["one_tile"] == 0 and pl["n_chunks"] > 1 and pl["items"] >= 5 * pl["grid"] and pl["grid"] == sms
    assert pl["bn"] == (128 if form.endswith("blocked") else 256) and pl["resident_b"] == 0


def _check_barely(pl, sms, tokens, form):
    assert pl["one_tile"] == 0 and sms < pl["items"] <= sms + 8 and pl["grid"] == sms and sms % pl["n_chunks"]
    assert pl["bn"] == (128 if form.endswith("blocked") else 256)


def _check_resident(pl, sms, tokens, form):
    assert pl["one_tile"] == 0 and pl["n_chunks"] == 1 and pl["m_tiles"] == sms + 1 and pl["resident_b"] == 1
    assert pl["bn"] == 48


def _check_streamed(pl, sms, tokens, form):
    assert pl["one_tile"] == 0 and pl["n_chunks"] == 1 and pl["m_tiles"] == sms + 1 and pl["resident_b"] == 0
    assert pl["num_kb"] > pl["stages"]


def _check_wraps(pl, sms, tokens, form):
    assert pl["one_tile"] == 1 and pl["resident_b"] == 0 and pl["num_kb"] == 44
    assert pl["num_kb"] > pl["stages"] and pl["num_kb"] % pl["stages"]


def _check_partial_k(pl, sms, tokens, form):
    _, ic, _, _ = _partial_k(sms, form)
    icp = up(ic, 32 if form.startswith("w4") else 16)
    assert icp % 128 and icp % 128 <= 96, "the last K block takes fewer than 4 k-steps"
    assert pl["num_kb"] == -(-icp // 128)


def _check_odd(pl, sms, tokens, form):
    assert tokens % 128 and pl["n_chunks"] * pl["bn"] > 1001, "ragged last m tile, columns past oc in the last n chunk"


def _check_bn16(pl, sms, tokens, form):
    assert pl["bn"] == 16 and pl["n_chunks"] == 1


CELLS = {
    "persistent_many_chunks": (_many_chunks, _check_many),
    "persistent_barely": (_barely, _check_barely),
    "persistent_one_chunk_resident_b": (_resident, _check_resident),
    "persistent_one_chunk_streamed_b": (_streamed, _check_streamed),
    "one_tile_ring_wraps_bs512": (_ring_wraps, _check_wraps),
    "partial_last_k_block_bs32": (_partial_k, _check_partial_k),
    "odd_oc_ragged_tiles": (_odd_oc, _check_odd),
    "bn16": (_bn16, _check_bn16),
}


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("cell", list(CELLS))
def test_linear_cell(backend, cell, form):
    sms = sm_count()
    shape, check_cell = CELLS[cell]
    tokens, ic, oc, bs = shape(sms, form)
    layer = Layer(backend, form, ic, oc, bs, seed=sum(map(ord, cell + form)))
    try:
        pl = layer.resize(tokens, variant_of(form, tokens))
        print(f"{cell} {form} (tokens {tokens}, ic {ic}, oc {oc}, bs {layer.bs}) on {sms} SMs: plan {pl}")
        assert pl["path"] == GEMM, pl
        max_bn = 128 if layer.bs else 256
        assert pl["bn"] == pick_bn(up(oc, 16), -(-tokens // 128), sms, max_bn), pl
        assert (pl["m_tiles"], pl["n_chunks"]) == (-(-tokens // 128), -(-up(oc, 16) // pl["bn"])), pl
        assert pl["items"] == pl["m_tiles"] * pl["n_chunks"] and pl["grid"] == min(pl["items"], sms), pl
        assert pl["one_tile"] == int(pl["items"] <= sms), pl
        try:
            check_cell(pl, sms, tokens, form)
        except AssertionError as e:
            raise AssertionError(f"{form} no longer lands in cell {cell}: plan {pl}") from e
        x = layer.inputs(tokens + ic)
        layer.check(x, layer.execute(x), f"{cell} {form}")
    finally:
        layer.destroy()


def pair_tokens(sms):
    """a CTA-pair launch with more work than pairs whose last 256-row pair tile holds 64 rows: its second CTA has none"""
    return 4096 + 64


@pytest.mark.parametrize("variant", [3, 0])
def test_linear_cell_cta_pair_empty_half(backend, variant):
    sms = sm_count()
    tokens = pair_tokens(sms)
    layer = Layer(backend, "w8", 2048, 6144, seed=7)
    try:
        pl = layer.resize(tokens, variant)
        print(f"cta_pair variant {variant} (tokens {tokens}, ic 2048, oc 6144) on {sms} SMs: plan {pl}")
        assert pl["path"] == PAIR and pl["bn"] == 256 and pl["m_tiles"] == -(-tokens // 256), pl
        assert 1 <= tokens % 256 <= 128, "the last pair tile's second CTA holds no rows"
        assert pl["items"] == pl["m_tiles"] * pl["n_chunks"] > pl["grid"] // 2 and pl["grid"] == sms // 2 * 2, pl
        assert (pl["one_tile"], pl["resident_b"]) == (0, 0), pl
        x = layer.inputs(11)
        layer.check(x, layer.execute(x), f"cta pair variant {variant}")
    finally:
        layer.destroy()


def _fresh(layer, tokens, x):
    """a new execution of the same layer resized once to tokens (auto variant): (plan, output)"""
    f = Layer.__new__(Layer)
    f.__dict__.update(layer.__dict__)
    f.h = layer.create()
    try:
        pl = f.resize(tokens, 0)
        return pl, f.execute(x)
    finally:
        f.destroy()


@pytest.mark.parametrize("form", FORMS)
def test_linear_one_execution_through_the_cells(backend, form):
    """one execution resized 4096 -> 9 -> 1 -> sms * 128 + 40 -> 300 tokens (auto variant), executed after each resize: the
    grow-only quantisation buffers and the tensor maps remade at each resize follow.  Plan and output equal those of a fresh
    execution, and the sampled rows equal the oracle"""
    sms = sm_count()
    layer = Layer(backend, form, 2048, 200, 64, seed=31)
    paths = []
    try:
        for tokens in (4096, 9, 1, sms * 128 + 40, 300):
            pl = layer.resize(tokens, 0)
            x = layer.inputs(tokens)
            y = layer.execute(x)
            fresh_pl, fresh_y = _fresh(layer, tokens, x)
            print(f"{form} resized to {tokens}: plan {pl}")
            assert pl == fresh_pl
            assert bool((y == fresh_y).all()), f"{tokens} tokens: the re-resized execution differs from a fresh one"
            if tokens > 1:
                layer.check(x, y, f"{form} at {tokens} tokens")
            paths.append(pl["path"])
    finally:
        layer.destroy()
    big = PAIR if form == "w8" else GEMM      # auto runs 8-bit per-channel layers of >= 256 tokens on the CTA pair
    assert paths == [big, GEMM, GEMV, big, big], paths


@pytest.mark.parametrize("form", ["w8", "w4"])
@pytest.mark.parametrize("tokens", [300, 5000])
def test_linear_gemm_y_misaligned(backend, form, tokens):
    """y 4 bytes past 8-byte alignment at an even oc (the GEMM's float2 stores would be misaligned): equal bit for bit to the
    aligned run, and to the oracle"""
    oc = 200
    layer = Layer(backend, form, 1024, oc, seed=tokens)
    try:
        pl = layer.resize(tokens, variant_of(form, tokens))
        assert pl["path"] == GEMM and oc % 2 == 0, pl
        x = layer.inputs(3)
        aligned = layer.execute(x)
        assert aligned.data_ptr() % 8 == 0
        shifted = layer.execute(x, y_offset=1)
        assert shifted.data_ptr() % 8 == 4
        assert bool((aligned == shifted).all()), "a misaligned y changed the output"
        layer.check(x, shifted, f"{form} misaligned y")
    finally:
        layer.destroy()


@pytest.mark.parametrize("form", FORMS)
def test_linear_plan_matches_execute(backend, form):
    """path -1 exactly where execute returns NOT_SUPPORT, for every variant at 1, 8, 9, 255 and 256 tokens: one token on the
    GEMM or the pair, 4-bit or blocked on the pair, the pair below 256 tokens, the GEMV above 8 tokens"""
    import torch
    layer = Layer(backend, form, 256, 64, 64, seed=2)
    try:
        f = (C.c_int * len(PLAN_FIELDS))(*([-7] * len(PLAN_FIELDS)))
        assert lib().mnnb200_linear_w8_plan(layer.h, f, len(f)) == NO_EXECUTION
        assert lib().mnnb200_linear_w8_plan(None, f, len(f)) == INVALID_VALUE
        assert list(f) == [-7] * len(PLAN_FIELDS)
        for tokens in (1, 8, 9, 255, 256):
            x = torch.zeros((tokens, 256), dtype=torch.float32, device="cuda")
            y = torch.zeros((tokens, 64), dtype=torch.float32, device="cuda")
            for variant in (0, 2, 3, 4):
                pl = layer.resize(tokens, variant)
                want = {0: GEMV if tokens <= 8 else PAIR if form == "w8" and tokens >= 256 else GEMM,
                        2: REFUSED if tokens == 1 else GEMM,
                        3: PAIR if form == "w8" and tokens >= 256 else REFUSED,
                        4: GEMV if tokens <= 8 else REFUSED}[variant]
                assert pl["path"] == want, (tokens, variant, pl)
                if want in (GEMV, REFUSED):
                    assert all(v == 0 for k, v in pl.items() if k != "path"), pl
                st = lib().mnnb200_linear_w8_execute(layer.h, C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()))
                assert st == (NOT_SUPPORT if want == REFUSED else 0), (tokens, variant, st)
        layer.backend.onSync()
        assert lib().mnnb200_conv_int8_set_variant(layer.h, 3) == 0
        assert lib().mnnb200_linear_w8_plan(layer.h, f, 2) == 0        # count limits what is written
        assert list(f)[:3] == ([PAIR, 64] if form == "w8" else [REFUSED, 0]) + [-7]
    finally:
        layer.destroy()
    conv = C.c_void_p()
    from mnn_b200._capi import ConvDesc
    d = ConvDesc(16, 16, 1, 1, 1, 1, 0, 0, 1, 1, 1, 0)
    w = np.zeros(256, np.float32)
    b = np.zeros(16, np.float32)
    assert lib().mnnb200_conv_f32_create(backend.runtime._h, C.byref(d), w.ctypes.data_as(C.c_void_p),
                                         b.ctypes.data_as(C.c_void_p), 0, C.byref(conv)) == 0
    try:
        f = (C.c_int * len(PLAN_FIELDS))()
        assert lib().mnnb200_linear_w8_plan(conv, f, len(f)) == INVALID_VALUE
    finally:
        lib().mnnb200_exec_destroy(conv)
