"""The fp32 MatMul / BatchMatMul through the C ABI (-m gpu), every output element against float64 on the CPU.

The kernel splits each fp32 operand into two TF32 parts, x = hi + lo, and sums a_hi*b_hi + a_hi*b_lo + a_lo*b_hi in fp32
accumulators.  Every output must lie within a worst-case model of that arithmetic (tolerance); a failure also reports what
plain TF32 (operands read with their low 13 mantissa bits dropped) would give.  Outputs are poisoned with NaN before each run
and sit between NaN guard cells, so an output left unwritten or a write outside C shows.  Covered: tile and N-chunk edges at
every transpose pair, the attention shapes of the transformer fixtures, probes that fail when either cross term is lost, every
broadcast form ShapeMatMul accepts, more than 65,535 batches and more than 2,097,120 operand rows, infinities and NaNs,
operands near FLT_MAX, unaligned pointers, rebinding, the sizes create refuses, and the Python backend's MatMulExecution."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import oracle as O

OK, NOT_SUPPORT, COMPUTE_SIZE_ERROR, INVALID_VALUE = 0, 2, 3, 5
GUARD = 64                    # NaN floats either side of C
MAX_BN = 128                  # the split kernel's widest n chunk


def lib():
    from mnn_b200 import _capi
    return _capi.lib()


def last_error():
    return lib().mnnb200_last_error().decode()


def arr(v):
    return (C.c_int * max(len(v), 1))(*v)


def tf32_trunc(a):
    """fp32 with the low 13 mantissa bits dropped: what a tensor core makes of an fp32 operand read as TF32"""
    return (np.ascontiguousarray(a, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_rna(a):
    """round fp32 to TF32 (10-bit mantissa, nearest, ties away): the hi part of the split"""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def pick_bn(n_padded, m_tiles, sm_count, max_bn=MAX_BN):
    """the create's n-chunk width (capi.cu pick_bn): equal chunks of at most max_bn columns, split further down to 32 columns
    while the M tiles alone leave SMs idle"""
    chunks = -(-n_padded // max_bn)
    if m_tiles * chunks < sm_count:
        want = min(sm_count // m_tiles, n_padded // 32)
        chunks = max(chunks, want)
    return (-(-n_padded // chunks) + 15) & ~15


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# Worst-case model of the split-TF32 product, per output element (tests/test_gpu_conv_f32.py::conv_tolerance with Kp = l padded
# to 8): a = a_hi + a_lo misses a by <= 2^-22 |a|, the dropped a_lo*b_lo is <= 2^-22 |a||b|, so the three products miss a*b by
# under 2^-20 |a||b|: 2^-20 S in all, S = |A| |B|.  Each of the 3 ceil(l / 8) wgmma k8 steps aligns its 8 products and the
# accumulator to the largest exponent and truncates, then truncates the normalised sum: (8 + 2) 2^-23 of its terms' magnitude
# sum, which S bounds.  The bias add rounds once, <= 2^-24 |acc + bias|, which 2^-23 (S + |bias|) covers.
def tolerance(s, l, bias=None):
    tau = 2.0 ** -20 + 3 * -(-l // 8) * (8 + 2) * 2.0 ** -23
    return tau * s + 2.0 ** -23 * (s + (0.0 if bias is None else np.abs(np.asarray(bias, np.float64))))


def logical(a, t):
    a = np.asarray(a, np.float64)
    return np.swapaxes(a, -1, -2) if t else a


def ref64(a, b, ta, tb, bias=None):
    """float64 (C, S) of op(A) op(B) (+ bias), numpy broadcasting the batch dims"""
    a64, b64 = logical(a, ta), logical(b, tb)
    ref = np.matmul(a64, b64) + (0.0 if bias is None else np.asarray(bias, np.float64))
    return ref, np.matmul(np.abs(a64), np.abs(b64))


def check(y, a, b, ta, tb, bias, what, ref=None, s=None):
    """every element within tolerance of float64; non-finite ones where float64 has them, infinities of the same sign"""
    if ref is None:
        ref, s = ref64(a, b, ta, tb, bias)
    y = np.asarray(y, np.float64)
    assert y.shape == ref.shape, (what, y.shape, ref.shape)
    fin = np.isfinite(ref)
    assert np.array_equal(np.isnan(y), np.isnan(ref)), f"{what}: NaN at {np.argwhere(np.isnan(y) != np.isnan(ref))[:4].tolist()}"
    inf = np.isinf(ref)
    assert np.array_equal(y[inf], ref[inf]) and np.isfinite(y[fin]).all(), f"{what}: infinities differ from float64"
    l = logical(a, ta).shape[-1]
    tol = tolerance(s, l, bias)
    err = np.where(fin, np.abs(np.where(fin, y, 0) - np.where(fin, ref, 0)), 0.0)
    over = err > np.where(fin, tol, np.inf)
    if over.any():
        i = tuple(np.argwhere(over)[0])
        plain = np.matmul(logical(tf32_trunc(a), ta), logical(tf32_trunc(b), tb)) + (0.0 if bias is None else np.asarray(bias, np.float64))
        pe = np.abs(np.where(fin, plain - ref, 0)) / np.where(fin, tol, np.inf)
        pytest.fail(f"{what}: {np.count_nonzero(over)} of {y.size} outputs over the bound; first at {i}: got {y[i]!r}, float64 "
                    f"{ref[i]!r}, |err| {err[i]:.3g} > {tol[i]:.3g}; worst at {float((err / np.where(fin, tol, np.inf)).max()):.2f} "
                    f"of its bound, plain TF32 would reach {float(pe.max()):.2f}")
    return float((err / np.where(fin, tol, np.inf)).max())


# ---- the C ABI ------------------------------------------------------------------------------------------------------------
def create(backend, batch, e, l, h, ta, tb):
    hdl = C.c_void_p()
    st = lib().mnnb200_matmul_create(backend.runtime._h, batch, e, l, h, int(ta), int(tb), 0, C.byref(hdl))
    assert st == OK, last_error()
    return hdl


def create_bc(backend, cd, ad, bd, e, l, h, ta, tb):
    hdl = C.c_void_p()
    st = lib().mnnb200_matmul_create_broadcast(backend.runtime._h, len(cd), arr(cd), arr(ad), arr(bd), e, l, h, int(ta), int(tb),
                                               C.byref(hdl))
    assert st == OK, last_error()
    return hdl


def dev(x, shift=0):
    """x on the device, `shift` floats past a 256-byte boundary"""
    import torch
    x = np.ascontiguousarray(x, np.float32)
    buf = torch.empty(x.size + shift, dtype=torch.float32, device="cuda")
    v = buf[shift:]
    v.copy_(torch.from_numpy(x.reshape(-1)))
    return v, buf


def execute(hdl, a, b, c_shape, bias=None, shift_a=0, shift_b=0, shift_c=0):
    """one execute on fresh device copies; C NaN-poisoned between NaN guards, which must stay NaN"""
    import torch
    da, _ka = dev(a, shift_a)
    db, _kb = dev(b, shift_b)
    dbias = None if bias is None else dev(bias)[0]
    n = int(np.prod(c_shape))
    cbuf = torch.full((n + 2 * GUARD + shift_c,), float("nan"), dtype=torch.float32, device="cuda")
    c = cbuf[GUARD + shift_c:GUARD + shift_c + n]
    st = lib().mnnb200_matmul_execute(hdl, C.c_void_p(da.data_ptr()), C.c_void_p(db.data_ptr()),
                                      None if dbias is None else C.c_void_p(dbias.data_ptr()), C.c_void_p(c.data_ptr()))
    assert st == OK, last_error()
    torch.cuda.synchronize()
    host = cbuf.cpu().numpy()
    assert np.isnan(host[:GUARD + shift_c]).all() and np.isnan(host[GUARD + shift_c + n:]).all(), "a write outside C"
    return host[GUARD + shift_c:GUARD + shift_c + n].reshape(c_shape)


def operands(rng, bd_a, bd_b, e, l, h, ta, tb, gen=None):
    gen = gen or (lambda s: rng.standard_normal(s).astype(np.float32))
    a = gen(tuple(bd_a) + ((l, e) if ta else (e, l)))
    b = gen(tuple(bd_b) + ((h, l) if tb else (l, h)))
    return a, b


def run_case(backend, bd, e, l, h, ta, tb, bias, rng, what):
    a, b = operands(rng, bd, bd, e, l, h, ta, tb)
    hdl = create(backend, int(np.prod(bd, dtype=np.int64)), e, l, h, ta, tb)
    try:
        y = execute(hdl, a, b, tuple(bd) + (e, h), bias)
    finally:
        lib().mnnb200_exec_destroy(hdl)
    return check(y, a, b, ta, tb, bias, what)


TRANS = [(False, False), (False, True), (True, False), (True, True)]
# (batch dims, e, l, h, bias): every l of {1, 3, 4, 5, 8, 9, 31, 33, 65, 200, 1000, 4096}, e of {1, 127, 128, 129, 300} (in batches
# of 2 or 3 where e % 128 != 0: a 128-row tile then spans two batches) and h of {1, 15, 16, 17, 255, 256, 257, 513}; bias on odd h
SHAPES = [((), 1, 1, 1, True), ((3,), 127, 3, 15, True), ((2,), 128, 4, 16, False), ((3,), 129, 5, 17, True),
          ((2,), 300, 8, 255, True), ((), 1, 9, 256, False), ((2,), 127, 31, 257, True), ((), 128, 33, 513, False),
          ((3,), 129, 65, 1, True), ((), 300, 200, 15, True), ((2,), 129, 1000, 17, False), ((), 127, 4096, 256, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("ta,tb", TRANS)
@pytest.mark.parametrize("si", range(len(SHAPES)))
def test_shapes_vs_float64(backend, si, ta, tb):
    bd, e, l, h, has_bias = SHAPES[si]
    rng = np.random.default_rng(100 * si + 2 * ta + tb)
    bias = rng.standard_normal(h).astype(np.float32) if has_bias else None
    run_case(backend, bd, e, l, h, ta, tb, bias, rng, f"{bd} e {e} l {l} h {h}")


def chunk_cases(sms):
    """for every n-chunk width the create can pick (16 ... 128), one (m_tiles, h) that picks it with a partial last chunk where
    the width allows more than one chunk"""
    cases = {}
    for m_tiles in range(1, 2 * sms + 1):
        for h in range(1, 700):
            bn = pick_bn((h + 15) & ~15, m_tiles, sms)
            chunks = -(-h // bn)
            good = chunks > 1 and h % bn != 0
            if bn not in cases or (good and not cases[bn][2]):
                cases[bn] = (m_tiles, h, good)
    return cases


@pytest.mark.gpu
def test_every_n_chunk_width(backend):
    """the create's rule picks each width from the SM count and the M tiles; each runs with a ragged last chunk (16 fits only
    h <= 16, one chunk)"""
    cases = chunk_cases(sm_count())
    assert sorted(cases) == list(range(16, MAX_BN + 1, 16)), sorted(cases)
    rng = np.random.default_rng(7)
    for bn, (m_tiles, h, good) in sorted(cases.items()):
        assert good or bn == 16, (bn, m_tiles, h)
        e = m_tiles * 128 - 3
        bias = rng.standard_normal(h).astype(np.float32) if h % 2 else None
        run_case(backend, (), e, 40, h, bn % 32 == 0, bn % 64 == 0, bias, rng, f"bn {bn}: e {e} h {h}")


# ---- accuracy where plain TF32 failed: the transformer fixtures' attention ---------------------------------------------------
def softmax_rows(rng, shape):
    x = np.exp(rng.standard_normal(shape) * 2)
    return (x / x.sum(-1, keepdims=True)).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("bd,e,l,h,tb,kind", [((2, 12), 128, 128, 64, False, "PV"), ((2, 3), 197, 197, 64, False, "PV"),
                                              ((2,), 64, 4096, 64, False, "PV"), ((2, 12), 128, 64, 128, True, "QK"),
                                              ((2, 3), 197, 64, 197, True, "QK")])
def test_attention_shapes(backend, bd, e, l, h, tb, kind):
    """PV: a softmax-probability left operand (non-negative: every dropped bit of plain TF32 errs the same way, so its error
    grows with l); QK^T with adjY.  Within the float64 bound, and within 1e-3 of the CPU backend's fp32 matmul"""
    rng = np.random.default_rng(e + l + h)
    a = softmax_rows(rng, bd + (e, l)) if kind == "PV" else rng.standard_normal(bd + (e, l)).astype(np.float32)
    b = rng.standard_normal(bd + ((h, l) if tb else (l, h))).astype(np.float32)
    hdl = create(backend, int(np.prod(bd)), e, l, h, False, tb)
    try:
        y = execute(hdl, a, b, bd + (e, h))
    finally:
        lib().mnnb200_exec_destroy(hdl)
    worst = check(y, a, b, False, tb, None, f"{kind} {bd} {e}x{l}x{h}")
    c32 = O.matmul_f32(a, b, False, tb)
    rel = float(np.abs(y - c32).max() / np.abs(c32).max())
    assert rel <= 1e-3, rel
    ref, s = ref64(a, b, False, tb)
    plain = np.matmul(tf32_trunc(a).astype(np.float64), logical(tf32_trunc(b), tb))
    print(f"{kind} {bd} {e}x{l}x{h}: worst output at {worst:.2f} of its bound, vs CPU fp32 {rel:.1e}; plain TF32 "
          f"{float(np.abs(plain - ref).max() / np.abs(ref).max()):.1e} of max|C|")
    if kind == "PV":        # plain TF32 breaks the per-element bound, or at deep l (where the bound is loose) the 1e-3 rule
        assert ((np.abs(plain - ref) > tolerance(s, l)).any() or np.abs(plain - ref).max() > 1e-3 * np.abs(ref).max()), \
            "plain TF32 would pass this case: it no longer shows the truncation"


def test_matmul_kernels_compile_without_spills(tmp_path):
    """(CPU) the split-TF32 and fp16 GEMM and their pack kernels compile for sm_90a without register spills"""
    from mnn_b200 import build as B
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-c", os.path.join(B.CSRC, "gemm_f16_wgmma.cu"), "-o", str(tmp_path / "k.o")] + B.NVCC_FLAGS + ["-Xptxas", "-v"]
    out = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    found, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            fn = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn:
            found[fn] = int(m.group(1)) + int(m.group(2))
    for k in ("gemm_f16_wgmma_kernelILb1E", "gemm_f16_wgmma_kernelILb0E", "pack_kmajor_f32_kernelIfE", "pack_kmajor_f16_kernelI6__halfE"):
        names = [n for n in found if k in n]
        assert names, f"{k} not compiled"
        assert all(found[n] == 0 for n in names), {n: found[n] for n in names}


# ---- split probes -----------------------------------------------------------------------------------------------------------
def probe_inputs(rng, probe, bd, e, l, h):
    """probe A: a = v + 2^-12 with v TF32-exact in [1, 2), b one-signed and TF32-exact: of the split terms only a_lo*b_hi carries
    the 2^-12.  Probe B is the mirror image, a TF32-exact and b = (u + 2^-12) 2^-6: only a_hi*b_lo carries it."""
    v = (1 + rng.integers(0, 1024, bd + (e, l)) / 1024).astype(np.float32)
    u = (1 + rng.integers(0, 1024, bd + (l, h)) / 1024).astype(np.float32)
    if probe == "A":
        return v + np.float32(2.0 ** -12), u * np.float32(2.0 ** -6)
    return v, (u + np.float32(2.0 ** -12)) * np.float32(2.0 ** -6)


PROBE_SHAPE = ((3,), 130, 64, 72)


def probe_reference(probe):
    bd, e, l, h = PROBE_SHAPE
    a, b = probe_inputs(np.random.default_rng(ord(probe)), probe, bd, e, l, h)
    ref, s = ref64(a, b, False, False)
    dropped = ref64(tf32_rna(a), b, False, False)[0] if probe == "A" else ref64(a, tf32_rna(b), False, False)[0]
    return a, b, ref, s, dropped


@pytest.mark.parametrize("probe", ["A", "B"])
def test_probe_inputs_separate_the_lost_term(probe):
    """(CPU) the probe's operands: the hi part is TF32-exact but for 2^-12 (scaled), the partner TF32-exact, and losing the lo
    term moves every output by more than twice its bound"""
    a, b, ref, s, dropped = probe_reference(probe)
    hi, lo = (a, b) if probe == "A" else (b, a)
    assert np.array_equal(tf32_rna(hi), hi - np.float32(2.0 ** -12 * (1 if probe == "A" else 2.0 ** -6)))
    assert np.array_equal(tf32_rna(lo), lo) and np.array_equal(tf32_trunc(lo), lo)
    assert (np.abs(ref - dropped) > 2 * tolerance(s, PROBE_SHAPE[2])).all()


@pytest.mark.gpu
@pytest.mark.parametrize("probe", ["A", "B"])
def test_split_probe(backend, probe):
    bd, e, l, h = PROBE_SHAPE
    a, b, ref, s, dropped = probe_reference(probe)
    hdl = create(backend, int(np.prod(bd)), e, l, h, False, False)
    try:
        y = execute(hdl, a, b, bd + (e, h))
    finally:
        lib().mnnb200_exec_destroy(hdl)
    worst = check(y, a, b, False, False, None, f"probe {probe}", ref, s)
    print(f"probe {probe}: worst output at {worst:.2f} of its bound; the lost term would move every output by at least "
          f"{float((np.abs(ref - dropped) / tolerance(s, l)).min()):.1f} bounds")


# ---- broadcast batches -----------------------------------------------------------------------------------------------------
# (A batch dims, B batch dims, e, l, h, ta, tb) as ShapeMatMul takes them (right-aligned; the shorter padded with 1s here)
BROADCAST = [
    ((3,), (1,), 20, 9, 24, False, False),                    # B broadcast, nd 1
    ((1,), (3,), 20, 9, 24, True, True),                      # A broadcast
    ((2, 1), (1, 3), 33, 16, 17, False, True),                # both, nd 2
    ((1, 1), (2, 3), 5, 8, 40, True, False),
    ((2, 1, 3), (2, 4, 1), 31, 12, 20, False, False),         # a 1 in the middle, nd 3
    ((1, 3, 1, 2), (2, 1, 4, 2), 17, 7, 9, True, True),       # nd 4
    ((2, 1, 2, 1, 1, 3, 1, 2), (1, 2, 2, 1, 2, 1, 1, 2), 9, 5, 11, False, True),   # nd 8
    ((4,), (1,), 50, 32, 48, False, False),                   # [B,S,D] x [D,E]
    ((1, 3), (2, 3), 40, 16, 40, False, False),               # [1,H,S,D] x [B,H,D,S]
    ((1, 1), (2, 3), 1, 24, 30, False, False),                # 1-D A [l] against [2,3,l,h]: e = 1
    ((2, 3), (1, 1), 30, 24, 1, True, True),                  # 1-D B [l] against [2,3,l,e]: h = 1, K-major B
]


@pytest.mark.gpu
@pytest.mark.parametrize("ci", range(len(BROADCAST)))
def test_broadcast_forms(backend, ci):
    ad, bd, e, l, h, ta, tb = BROADCAST[ci]
    cd = tuple(max(x, y) for x, y in zip(ad, bd))
    rng = np.random.default_rng(ci + 40)
    a, b = operands(rng, ad, bd, e, l, h, ta, tb)
    hdl = create_bc(backend, cd, ad, bd, e, l, h, ta, tb)
    try:
        y = execute(hdl, a, b, cd + (e, h))
    finally:
        lib().mnnb200_exec_destroy(hdl)
    check(y, a, b, ta, tb, None, f"{ad} x {bd}")


@pytest.mark.gpu
@pytest.mark.parametrize("ta,tb", TRANS)
def test_no_broadcast_equals_plain_create(backend, ta, tb):
    """with no dim to broadcast, create_broadcast makes mnnb200_matmul_create's execution: the same bits"""
    bd, e, l, h = (2, 3), 70, 45, 50
    rng = np.random.default_rng(2 * ta + tb)
    a, b = operands(rng, bd, bd, e, l, h, ta, tb)
    bias = rng.standard_normal(h).astype(np.float32)
    h1, h2 = create_bc(backend, bd, bd, bd, e, l, h, ta, tb), create(backend, 6, e, l, h, ta, tb)
    try:
        y1, y2 = execute(h1, a, b, bd + (e, h), bias), execute(h2, a, b, bd + (e, h), bias)
    finally:
        lib().mnnb200_exec_destroy(h1)
        lib().mnnb200_exec_destroy(h2)
    assert np.array_equal(y1.view(np.uint32), y2.view(np.uint32))
    check(y1, a, b, ta, tb, bias, "no broadcast")


# ---- sizes past the launch grid's y / z limits ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("ta,tb", TRANS)
@pytest.mark.parametrize("form", ["batched", "a_broadcast", "b_broadcast"])
def test_more_than_65535_batches(backend, form, ta, tb):
    n, e, l, h = 70000, 4, 8, 4
    ad, bd = {"batched": ((n,), (n,)), "a_broadcast": ((1,), (n,)), "b_broadcast": ((n,), (1,))}[form]
    rng = np.random.default_rng(len(form) + 2 * ta + tb)
    a, b = operands(rng, ad, bd, e, l, h, ta, tb)
    hdl = create(backend, n, e, l, h, ta, tb) if form == "batched" else create_bc(backend, (n,), ad, bd, e, l, h, ta, tb)
    try:
        y = execute(hdl, a, b, (n, e, h))
    finally:
        lib().mnnb200_exec_destroy(hdl)
    check(y, a, b, ta, tb, None, f"{form} {n} batches")


@pytest.mark.gpu
@pytest.mark.parametrize("side,t", [("A", False), ("A", True), ("B", False), ("B", True)])
def test_operand_of_more_than_2097120_rows(backend, side, t):
    """one operand of 2.2M rows (e for A, h for B), l = 8: its pack covers 68,750 32-row tiles"""
    rows = 2_200_000
    e, l, h = (rows, 8, 4) if side == "A" else (3, 8, rows)
    ta, tb = (t, False) if side == "A" else (False, t)
    rng = np.random.default_rng(rows + t)
    a, b = operands(rng, (), (), e, l, h, ta, tb)
    hdl = create(backend, 1, e, l, h, ta, tb)
    try:
        y = execute(hdl, a, b, (e, h))
    finally:
        lib().mnnb200_exec_destroy(hdl)
    check(y, a, b, ta, tb, None, f"{side} of {rows} rows")


# ---- special values ---------------------------------------------------------------------------------------------------------
NAN_LOW = np.array([0x7F800001, 0xFF801FFF], np.uint32).view(np.float32)   # NaNs whose payload lies in the 13 bits TF32 drops


def partners(rng, shape):
    """finite operands with zeros and TF32-exact values among them (an infinity times those is NaN and +-Inf in fp32)"""
    x = rng.standard_normal(shape).astype(np.float32)
    x.flat[::7] = 0.0
    x.flat[3::7] = np.float32(1.0) * np.sign(x.flat[3::7])
    return x


# a row of A or a column of B meets mixed-sign partners along k (NaN outputs); a column of A, a row of B or one element meets
# one partner per output: +-Inf, or NaN where the partner is 0
MIXED = {"a_col_inf", "a_one_inf", "b_row_inf", "b_one_inf", "a_b_inf_apart"}
SPECIAL = ["a_row_inf", "a_col_inf", "a_one_inf", "a_nan_low", "b_row_inf", "b_col_inf", "b_one_inf", "b_nan_low", "a_b_inf_apart"]


def special_operands(rng, case, e, l, h):
    """A [e][l], B [l][h] (logical).  Infinities in A and in B never share a k: Inf * Inf is the one product the split does
    not give as fp32 does (see split_tf32)."""
    a, b = partners(rng, (e, l)), partners(rng, (l, h))
    side, kind = case[0], case[2:]
    x = a if side == "a" else b
    r, k = (5, 3) if side == "a" else (3, 7)       # a row / column of x
    if kind == "row_inf":
        x[r, :] = np.where(rng.random(x.shape[1]) < 0.5, -np.inf, np.inf)
    elif kind == "col_inf":
        x[:, k] = np.where(rng.random(x.shape[0]) < 0.5, -np.inf, np.inf)
    elif kind == "one_inf":
        x[r, k], x[r + 1, k + 1] = np.inf, -np.inf
    elif kind == "nan_low":                        # one element, and one output row (A) or column (B)
        x[r, k] = NAN_LOW[0]
        if side == "a":
            x[r + 2, :] = NAN_LOW[1]
        else:
            x[:, k + 2] = NAN_LOW[1]
    elif case == "a_b_inf_apart":
        a[:, 2] = np.inf
        b[5, :] = -np.inf
        a[4, 9] = -np.inf
    return a, b


def ref_elementwise(a, b):
    """float64 C and S summing a_ik * b_kj explicitly (IEEE special values, no BLAS)"""
    a64, b64 = np.asarray(a, np.float64), np.asarray(b, np.float64)
    with np.errstate(invalid="ignore"):
        return (a64[:, :, None] * b64[None, :, :]).sum(1), (np.abs(a64)[:, :, None] * np.abs(b64)[None, :, :]).sum(1)


@pytest.mark.gpu
@pytest.mark.parametrize("ta,tb", [(False, False), (True, True)])
@pytest.mark.parametrize("case", SPECIAL)
def test_special_values(backend, case, ta, tb):
    """infinities of either sign in single rows, columns and elements of A and B, against zeros and TF32-exact partners, and
    NaNs with only low payload bits: every non-finite output where float64 has one (infinities with its sign), every finite one
    within the bound"""
    e, l, h = 40, 24, 36
    rng = np.random.default_rng(SPECIAL.index(case))
    a, b = special_operands(rng, case, e, l, h)
    ref, s = ref_elementwise(a, b)
    assert (~np.isfinite(ref)).any()
    if case in MIXED:
        assert np.isinf(ref).any() and np.isnan(ref).any(), "the case no longer has both infinite and NaN outputs"
    sa, sb = (a.T.copy() if ta else a), (b.T.copy() if tb else b)
    hdl = create(backend, 1, e, l, h, ta, tb)
    try:
        y = execute(hdl, sa, sb, (e, h))
    finally:
        lib().mnnb200_exec_destroy(hdl)
    check(y, sa, sb, ta, tb, None, case, ref, np.where(np.isfinite(s), s, 0))
    if case.endswith("nan_low"):
        plain = np.matmul(tf32_trunc(a).astype(np.float64), tf32_trunc(b).astype(np.float64))
        assert np.isinf(plain).any(), "plain TF32 reads these NaNs as infinities"


@pytest.mark.gpu
@pytest.mark.parametrize("big", ["A", "B"])
def test_near_flt_max(backend, big):
    """operands of the top binades, FLT_MAX and values that round to infinity as TF32 among them, against partners of at most
    2^-8 / l at l = 6: every output finite and within the bound"""
    e, l, h = 33, 6, 20
    rng = np.random.default_rng(ord(big))
    fmax = np.finfo(np.float32).max
    huge = (fmax * rng.uniform(0.5, 1.0, (e, l) if big == "A" else (l, h))).astype(np.float32)
    huge *= np.where(rng.random(huge.shape) < 0.5, -1, 1).astype(np.float32)
    huge.flat[0], huge.flat[1], huge.flat[2] = fmax, -fmax, np.float32(2 - 2.0 ** -11) * np.float32(2.0 ** 127)
    assert np.isinf(tf32_rna(huge)).sum() >= 3
    small = (rng.uniform(-1, 1, (l, h) if big == "A" else (e, l)) * 2.0 ** -8 / l).astype(np.float32)
    a, b = (huge, small) if big == "A" else (small, huge)
    hdl = create(backend, 1, e, l, h, False, False)
    try:
        y = execute(hdl, a, b, (e, h))
    finally:
        lib().mnnb200_exec_destroy(hdl)
    ref, s = ref_elementwise(a, b)
    assert np.isfinite(ref).all()
    check(y, a, b, False, False, None, f"near FLT_MAX in {big}", ref, s)


# ---- pointers --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("ta,tb", TRANS)
def test_unaligned_pointers(backend, ta, tb):
    """C one float past an 8-byte boundary with even h (no float2 store may land there), and A and B 4 bytes past 16-byte
    alignment"""
    bd, e, l, h = (2,), 150, 37, 72
    rng = np.random.default_rng(60 + 2 * ta + tb)
    a, b = operands(rng, bd, bd, e, l, h, ta, tb)
    bias = rng.standard_normal(h).astype(np.float32)
    hdl = create(backend, 2, e, l, h, ta, tb)
    try:
        y = execute(hdl, a, b, bd + (e, h), bias, shift_a=1, shift_b=3, shift_c=1)
    finally:
        lib().mnnb200_exec_destroy(hdl)
    check(y, a, b, ta, tb, bias, "unaligned")


@pytest.mark.gpu
def test_rebinds_between_runs(backend):
    """one execution run on three sets of buffers, each with other data: every run reads its own operands"""
    bd, e, l, h = (2,), 150, 64, 72
    rng = np.random.default_rng(21)
    hdl = create(backend, 2, e, l, h, False, True)
    try:
        for shift in (0, 0, 1):
            a, b = operands(rng, bd, bd, e, l, h, False, True)
            bias = rng.standard_normal(h).astype(np.float32)
            check(execute(hdl, a, b, bd + (e, h), bias, shift, shift, 2 * shift), a, b, False, True, bias, f"rebound {shift}")
    finally:
        lib().mnnb200_exec_destroy(hdl)


# ---- refusals --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals_launch_nothing(backend):
    """sizes beyond the kernel's 32-bit row, byte and work indices return NOT_SUPPORT from create, too many broadcast batches
    INVALID_VALUE, before anything is allocated or launched"""
    L, rt = lib(), backend.runtime._h
    before = L.mnnb200_launch_count()
    hdl = C.c_void_p()
    refused = [
        (L.mnnb200_matmul_create(rt, 70000, 20000, 8, 4, 0, 0, 0, C.byref(hdl)), NOT_SUPPORT),        # A: 1.4e9 rows per plane
        (L.mnnb200_matmul_create(rt, 70000, 4, 8, 20000, 0, 0, 0, C.byref(hdl)), NOT_SUPPORT),        # B
        (L.mnnb200_matmul_create(rt, 1, 4, (1 << 29) + 1, 4, 0, 0, 0, C.byref(hdl)), NOT_SUPPORT),    # 2^31 bytes per row
        (L.mnnb200_matmul_create(rt, 1, 1 << 29, 8, 1 << 29, 0, 0, 1, C.byref(hdl)), NOT_SUPPORT),    # 2^37 work items (fp16)
        (L.mnnb200_matmul_create_broadcast(rt, 2, arr((65536, 65536)), arr((65536, 1)), arr((1, 65536)), 1, 8, 1, 0, 0,
                                           C.byref(hdl)), INVALID_VALUE),                           # 2^32 output batches
        (L.mnnb200_matmul_create_broadcast(rt, 2, arr((40000, 40000)), arr((40000, 1)), arr((1, 40000)), 1, 8, 1, 0, 0,
                                           C.byref(hdl)), NOT_SUPPORT),                             # 1.6e9 batches: 2 planes
    ]
    assert [st for st, _ in refused] == [want for _, want in refused], last_error()
    assert not hdl.value
    assert L.mnnb200_launch_count() == before


# ---- the Python backend's MatMulExecution ----------------------------------------------------------------------------------
MIRROR = [  # (A shape, B shape, transpose_a, transpose_b): stored shapes
    ((2, 3, 20, 9), (2, 3, 9, 24), False, False),   # batched
    ((4, 30, 16), (16, 24), False, False),          # 3-D x 2-D: [B,S,D] x [D,E]
    ((24, 30), (2, 3, 24, 17), True, False),        # 2-D x 4-D
    ((1, 3, 20, 8), (2, 1, 20, 8), False, True),    # both broadcast
    ((9,), (2, 9, 7), False, False),                # 1-D A
    ((2, 9, 5), (9,), True, True),                  # 1-D B (transpose_b ignored)
    ((9,), (9,), False, False),                     # both 1-D
]


def mirror_run(backend, a, b, ta, tb):
    import torch
    from mnn_b200.backend import Op, Tensor
    d = backend.runtime.device
    ta_, tb_ = Tensor(a.shape, "float", None, torch.from_numpy(a).to(d)), Tensor(b.shape, "float", None, torch.from_numpy(b).to(d))
    y = Tensor((1,), "float")
    ex = backend.onCreate([ta_, tb_], [y], Op(type="BatchMatMul", extra=dict(transpose_a=ta, transpose_b=tb)))
    assert ex is not None
    st = ex.onResize([ta_, tb_], [y])
    if st:
        return st, None
    backend.onAcquire(y)
    y.data.fill_(float("nan"))
    assert ex.onExecute([ta_, tb_], [y]) == 0
    backend.onSync()
    return 0, y.data.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("mi", range(len(MIRROR)))
def test_python_matmul_execution(backend, mi):
    """ShapeMatMul's output shape and values (numpy's matmul rule, which squeezes 1-D operands the same way)"""
    sa, sb, ta, tb = MIRROR[mi]
    rng = np.random.default_rng(mi + 70)
    a, b = rng.standard_normal(sa).astype(np.float32), rng.standard_normal(sb).astype(np.float32)
    st, y = mirror_run(backend, a, b, ta, tb)
    assert st == 0, last_error()
    a64 = np.asarray(a, np.float64)
    a64 = np.swapaxes(a64, -1, -2) if ta and a.ndim > 1 else a64
    b64 = np.asarray(b, np.float64)
    b64 = np.swapaxes(b64, -1, -2) if tb and b.ndim > 1 else b64
    ref, s = np.matmul(a64, b64), np.matmul(np.abs(a64), np.abs(b64))
    ref, s = (ref.reshape(1), s.reshape(1)) if ref.ndim == 0 else (ref, s)
    assert y.shape == ref.shape, (y.shape, ref.shape)
    assert (np.abs(y - ref) <= tolerance(s, a64.shape[-1])).all()


@pytest.mark.gpu
@pytest.mark.parametrize("sa,sb,ta,tb,f16,want", [((2, 5, 9), (3, 9, 4), False, False, False, NOT_SUPPORT),   # 2 against 3
                                                  ((5, 9), (8, 4), False, False, False, COMPUTE_SIZE_ERROR),
                                                  ((2, 5, 9), (1, 9, 4), False, False, True, NOT_SUPPORT),    # fp16 broadcast
                                                  ((9,), (8,), False, False, False, COMPUTE_SIZE_ERROR)])
def test_python_matmul_execution_refusals(backend, sa, sb, ta, tb, f16, want):
    dt = np.float16 if f16 else np.float32
    st, _ = mirror_run(backend, np.zeros(sa, dt), np.zeros(sb, dt), ta, tb)
    assert st == want
