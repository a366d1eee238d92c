"""Float MatMul / BatchMatMul (SURVEY a9): oracle pinned on the reference CPU backend and on a committed fixture; the
wgmma f16 / split-TF32 path (-m gpu) within BASELINE's 1e-3 (max|d| / max|ref|) and every element within a model of its
arithmetic against float64."""
import os

import numpy as np
import pytest

from oracle import oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden", "matmul_golden.npz")
needs_ref = pytest.mark.skipif(not O.have_reference(), reason="oracle/_ref not built")
# (batch dims, e, l, h, transpose_a, transpose_b): attention QK^T / PV of Qwen-1.8B (16 heads x 128), plus ragged shapes
CASES = [((2, 4), 64, 128, 64, False, True), ((3,), 64, 64, 128, False, False), ((), 37, 53, 29, False, False),
         ((), 40, 24, 56, True, False), ((2,), 33, 72, 17, True, True), ((), 1, 200, 300, False, True)]


def make(rng, bd, e, l, h, ta, tb, positive=False):
    sa = bd + ((l, e) if ta else (e, l))
    sb = bd + ((h, l) if tb else (l, h))
    a = rng.uniform(0 if positive else -1, 1, sa).astype(np.float32)
    b = rng.uniform(-1, 1, sb).astype(np.float32)
    return a, b


def test_oracle_vs_golden_fixture():
    g = np.load(GOLD)
    for i in range(int(g["ncase"])):
        y = O.matmul_f32(g[f"m{i}_a"], g[f"m{i}_b"], bool(g[f"m{i}_ta"]), bool(g[f"m{i}_tb"]))
        ref = g[f"m{i}_y"]
        assert y.shape == ref.shape and np.abs(y - ref).max() <= 1e-5 * np.abs(ref).max()


@needs_ref
@pytest.mark.reference
def test_oracle_vs_live_reference():
    rng = np.random.default_rng(3)
    for bd, e, l, h, ta, tb in CASES[:4]:
        a, b = make(rng, bd, e, l, h, ta, tb)
        ref = O.ref_matmul(a, b, ta, tb)
        assert np.abs(O.matmul_f32(a, b, ta, tb) - ref).max() <= 1e-5 * np.abs(ref).max()


def run_matmul(backend, a, b, ta, tb, bias=None):
    """a, b: fp32 or fp16 host arrays (fp16 operands select the f16 wgmma kernel)"""
    import torch
    from mnn_b200.backend import Op, Tensor
    dev = backend.runtime.device
    ta_ = Tensor(a.shape, "float", None, torch.from_numpy(a).to(dev))
    tb_ = Tensor(b.shape, "float", None, torch.from_numpy(b).to(dev))
    y = Tensor((1,), "float")
    ex = backend.onCreate([ta_, tb_], [y], Op(type="BatchMatMul" if a.ndim > 2 else "MatMul", bias=bias,
                                              extra=dict(transpose_a=ta, transpose_b=tb)))
    assert ex is not None and ex.onResize([ta_, tb_], [y]) == 0
    backend.onAcquire(y)
    y.data.fill_(float("nan"))
    assert ex.onExecute([ta_, tb_], [y]) == 0
    backend.onSync()
    return y.data.cpu().numpy()


@pytest.mark.gpu
def test_gpu_vs_golden_and_oracle(backend):
    g = np.load(GOLD)
    for i in range(int(g["ncase"])):
        y = run_matmul(backend, g[f"m{i}_a"], g[f"m{i}_b"], bool(g[f"m{i}_ta"]), bool(g[f"m{i}_tb"]))
        ref = g[f"m{i}_y"]
        assert y.shape == ref.shape and not np.isnan(y).any()
        assert np.abs(y - ref).max() <= 1e-3 * np.abs(ref).max(), f"case {i}: {np.abs(y - ref).max() / np.abs(ref).max()}"


@pytest.mark.gpu
@pytest.mark.parametrize("bd,e,l,h,ta,tb", [((8, 16), 512, 128, 512, False, True), ((8, 16), 512, 512, 128, False, False),
                                            ((), 300, 1000, 260, False, False), ((2,), 130, 520, 40, True, True)])
def test_gpu_attention_shapes_vs_oracle(backend, bd, e, l, h, ta, tb):
    """BASELINE configs[3] attention BMM shapes (8 x 16 heads: [512,128]x[128,512] and [512,512]x[512,128]); the second
    with a non-negative left operand (softmax probabilities), the worst case for one-sided rounding."""
    rng = np.random.default_rng(e + l)
    a, b = make(rng, bd, e, l, h, ta, tb, positive=(l == 512))
    bias = rng.uniform(-1, 1, h).astype(np.float32) if not bd else None
    y = run_matmul(backend, a, b, ta, tb, bias)
    ref = O.matmul_f32(a, b, ta, tb, bias)
    assert np.abs(y - ref).max() <= 1e-3 * np.abs(ref).max(), np.abs(y - ref).max() / np.abs(ref).max()


# ---- every element against float64 ------------------------------------------------------------------------------------
# Worst-case model of the tensor-core accumulator: each wgmma k-step adds K products (K = 16 fp16 / 8 tf32) to the fp32
# accumulator by aligning all K + 1 terms to the largest exponent and truncating, then truncating the normalised sum to
# 24 bits.  Each step then errs by at most (K + 2) 2^-23 times the magnitude sum of its terms, which is at most
# S = sum_k |a_ik| |b_kj|; over ceil(l / K) steps the accumulation error is <= (K + 2) ceil(l / K) 2^-23 S.
# fp16 operands: products of 11-bit significands are exact in fp32, so that is all.  fp32 operands are split into TF32 parts,
# a = a_hi + a_lo, and summed as a_hi b_hi + a_hi b_lo + a_lo b_hi (three k8 steps per 8 products): the split misses a by
# <= 2^-22 |a|, the dropped a_lo b_lo is <= 2^-22 |a||b|, under 2^-20 S in all (tests/test_gpu_matmul_f32.py::tolerance).
# The epilogue's bias add rounds once: <= 2^-24 |C + bias|, which 2^-23 (S + |bias|) covers.
def tolerance(a64, b64, l, f16, bias):
    s = np.matmul(np.abs(a64), np.abs(b64))
    tau = 18 * -(-l // 16) * 2.0 ** -23 if f16 else 2.0 ** -20 + 3 * -(-l // 8) * 10 * 2.0 ** -23
    return tau * s + 2.0 ** -23 * (s + (0.0 if bias is None else np.abs(bias.astype(np.float64))))


def check_vs_float64(y, a, b, ta, tb, bias):
    f16 = a.dtype == np.float16
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    if ta:
        a64 = np.swapaxes(a64, -1, -2)
    if tb:
        b64 = np.swapaxes(b64, -1, -2)
    ref = np.matmul(a64, b64) + (0.0 if bias is None else bias.astype(np.float64))
    assert y.shape == ref.shape and not np.isnan(y).any()
    err, tol = np.abs(y - ref), tolerance(a64, b64, a64.shape[-1], f16, bias)
    assert (err <= tol).all(), f"{np.count_nonzero(err > tol)} elements over; worst excess {(err - tol).max():.3g}"
    # the ABI's accuracy contract against the CPU backend's fp32 matmul (O.matmul_f32 is pinned on it above)
    c32 = O.matmul_f32(a.astype(np.float32), b.astype(np.float32), ta, tb, bias)
    assert np.abs(y - c32).max() <= 1e-3 * np.abs(c32).max()


# (batch dims, e, l, h, bias): l in {1, 3, 4, 8, 9, 65, 200}; batches with e % 128 != 0 (a 128-row tile spans two batches);
# h > 256 (several N chunks); odd h with bias (the scalar store of the last column); e = 1
MM_SHAPES = [((), 37, 1, 29, True), ((), 64, 3, 40, False), ((3,), 200, 4, 24, False), ((2,), 130, 8, 300, False),
             ((), 1, 9, 17, True), ((2,), 150, 65, 33, True), ((), 129, 200, 513, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("f16", [False, True], ids=["tf32", "f16"])
@pytest.mark.parametrize("ta,tb", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("si", range(len(MM_SHAPES)))
def test_gpu_matmul_vs_float64(backend, si, ta, tb, f16):
    bd, e, l, h, has_bias = MM_SHAPES[si]
    rng = np.random.default_rng(si * 8 + ta * 4 + tb * 2 + f16)
    a, b = make(rng, bd, e, l, h, ta, tb)
    if f16:
        a, b = a.astype(np.float16), b.astype(np.float16)
    bias = rng.uniform(-1, 1, h).astype(np.float32) if has_bias else None
    check_vs_float64(run_matmul(backend, a, b, ta, tb, bias), a, b, ta, tb, bias)


@pytest.mark.gpu
def test_gpu_matmul_rebinds_and_packs_misaligned(backend):
    """One execution run three times: on aligned K-major operands, on other aligned buffers (every run must read its own
    operands), and on operands that start one float past a 16-byte boundary."""
    import torch
    from mnn_b200.backend import Op, Tensor
    bd, e, l, h = (2,), 150, 64, 72          # ta = 0, tb = 1, l % 4 == 0: both operands K-major and aligned
    rng = np.random.default_rng(21)
    bias = rng.uniform(-1, 1, h).astype(np.float32)

    def dev(x, shift):
        buf = torch.empty(x.size + shift, dtype=torch.float32, device=backend.runtime.device)
        v = buf[shift:].view(x.shape)
        v.copy_(torch.from_numpy(x))
        assert (v.data_ptr() % 16 == 0) == (shift == 0)
        return v

    ex, y, seen = None, Tensor((1,), "float"), []
    for shift in (0, 0, 1):
        a, b = make(rng, bd, e, l, h, False, True)
        ta_, tb_ = Tensor(a.shape, "float", None, dev(a, shift)), Tensor(b.shape, "float", None, dev(b, shift))
        assert ta_.data.data_ptr() not in [t.data.data_ptr() for t in seen]
        seen.append(ta_)
        if ex is None:
            ex = backend.onCreate([ta_, tb_], [y], Op(type="BatchMatMul", bias=bias, extra=dict(transpose_a=False,
                                                                                                   transpose_b=True)))
            assert ex is not None and ex.onResize([ta_, tb_], [y]) == 0
            backend.onAcquire(y)
        y.data.fill_(float("nan"))
        assert ex.onExecute([ta_, tb_], [y]) == 0
        backend.onSync()
        check_vs_float64(y.data.cpu().numpy(), a, b, False, True, bias)
