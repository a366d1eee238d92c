"""The LLM linear layer with 4-bit weights (MNN-LLM's default --quant_bit 4 export) on the GPU (-m gpu):
mnnb200_linear_w4_create_blocked keeps only the packed nibbles on the device and runs on the existing GEMM (>= 9 tokens, the
nibbles expanded in shared memory) and GEMV (<= 8 tokens, expanded in registers) kernel instantiations.  Every output must equal
W.linear_w4_dynamic_blocks bit for bit, NaN-poisoned outputs included; the GEMV and the GEMM agree bit for bit for 2..8 tokens.
The plugin cases drive the reference's own Executor through libmnn_b200_plugin.so (skipped without oracle/_ref)."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import w4_oracle as W
from tests.test_gpu_block_linear import PLUGIN, run_on_plugin, status_codes
from tests.test_gpu_dispatch import (GOLDEN_TOL, check_linear, create_linear, golden_cases, golden_check,
                                     golden_check_profiled_in_child, linear_data, profile_golden_cases, run_linear)


@pytest.mark.gpu
def test_w4_linear_golden_cases(backend):
    golden_check(backend, 4)


@pytest.mark.gpu
def test_w4_linear_launches_listed_kernels():
    """the golden cases again, every variant under torch.profiler: only instantiations KERNEL_TESTS lists are launched (in a
    child process, for the reason test_block_linear_launches_listed_kernels gives)"""
    golden_check_profiled_in_child("tests.test_gpu_w4_linear")


SWEEP = [  # (tokens, ic, oc, bs (0: per channel), asym, bias, relu, relu6)
    (1, 256, 40, 32, True, True, False, False), (1, 5504, 264, 64, True, True, False, False), (1, 2048, 33, 128, False, False, False, True),
    (1, 1024, 300, 256, True, False, True, False), (1, 1024, 16, 512, True, True, False, False), (1, 2048, 2100, 0, True, True, False, False),
    (1, 2048, 8500, 64, False, True, False, False),
    (2, 2048, 2100, 64, True, True, False, False), (2, 512, 33, 32, False, True, False, False), (3, 1000, 70, 0, False, True, False, False),
    (4, 4096, 520, 128, True, False, False, True), (5, 5504, 48, 64, True, False, True, False), (6, 768, 40, 256, False, False, False, False),
    (7, 1024, 100, 0, True, True, False, False), (8, 1024, 520, 128, True, True, False, False), (8, 2048, 4300, 64, False, True, False, False),
    (9, 256, 33, 32, True, True, False, False), (9, 5504, 200, 64, True, True, False, False), (9, 1536, 70, 0, True, False, False, True),
    (100, 2048, 2048, 128, True, False, False, False), (100, 1024, 40, 256, False, True, False, True), (100, 2048, 130, 0, True, True, True, False),
    (256, 5504, 600, 64, True, True, False, False), (256, 640, 1000, 32, True, True, False, False), (256, 2048, 2048, 0, False, True, False, False),
    (512, 2048, 2048, 64, True, True, False, False), (512, 4096, 264, 512, False, False, False, False), (512, 1024, 3000, 0, True, False, False, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("tokens,ic,oc,bs,asym,has_bias,relu,relu6", SWEEP)
def test_w4_linear_sweep(backend, tokens, ic, oc, bs, asym, has_bias, relu, relu6):
    rng = np.random.default_rng(tokens * 7919 + ic * 31 + oc + bs)
    x, wp, alpha, wzero, bias = linear_data(rng, tokens, ic, oc, asym, has_bias, bits=4, bs=bs)
    check_linear(backend, x, wp, alpha, wzero, bias, 4, relu=relu, relu6=relu6)


@pytest.mark.gpu
@pytest.mark.parametrize("tokens,bs", [(1, 64), (3, 0), (20, 64), (300, 128)])
def test_w4_linear_zero_row_misaligned(backend, tokens, bs):
    """an all-zero token row (the amax < 1e-7 / range <= 1e-7 branches) and x 4 bytes past 16-byte alignment"""
    rng = np.random.default_rng(5 + tokens)
    x, wp, alpha, wzero, bias = linear_data(rng, tokens, 1024, 72, True, True, bits=4, bs=bs)
    x[tokens // 2] = 0
    check_linear(backend, x, wp, alpha, wzero, bias, 4, misalign=True)


@pytest.mark.gpu
def test_w4_linear_gemv_equals_gemm_and_refusals(backend):
    import torch
    from mnn_b200 import _capi
    lib = _capi.lib()
    inval, nsup = status_codes()
    rng = np.random.default_rng(3)
    ic, oc = 512, 96
    for tokens in range(2, 9):       # GEMV (variant 4) and GEMM (variant 2): identical bits
        for bs in (64, 0):
            x, wp, alpha, wzero, bias = linear_data(rng, tokens, ic, oc, True, True, bits=4, bs=bs)
            res = run_linear(backend, x, wp, alpha, wzero, bias, (4, 2), 4)
            assert np.array_equal(res[4][0], res[2][0]), f"{tokens} tokens, bs {bs}: GEMV and GEMM differ"
    x, wp, alpha, wzero, bias = linear_data(rng, 300, ic, oc, True, True, bits=4, bs=64)
    st, h = create_linear(backend, ic, oc, wp, alpha, wzero, bias, 4)
    assert st == 0
    try:
        xd = torch.from_numpy(x).cuda()
        yd = torch.empty((300, oc), dtype=torch.float32, device="cuda")
        assert lib.mnnb200_linear_w8_resize(h, 300) == 0
        assert lib.mnnb200_conv_int8_set_variant(h, 3) == 0          # the CTA-pair GEMM takes 8-bit weights only
        assert lib.mnnb200_linear_w8_execute(h, C.c_void_p(xd.data_ptr()), C.c_void_p(yd.data_ptr())) == nsup
        assert lib.mnnb200_linear_w8_resize(h, 1) == 0
        assert lib.mnnb200_conv_int8_set_variant(h, 2) == 0          # one token on a forced GEMM
        assert lib.mnnb200_linear_w8_execute(h, C.c_void_p(xd.data_ptr()), C.c_void_p(yd.data_ptr())) == nsup
    finally:
        lib.mnnb200_exec_destroy(h)
    wp = np.zeros(oc * ic // 2, np.uint8)
    for blocks, want in ((0, inval), (-1, inval), (3, inval), (ic // 16, nsup), (1, 0)):
        al = np.ones((oc, max(blocks, 1)), np.float32)
        st, h = create_linear(backend, ic, oc, wp, al, bits=4, blocks=blocks)
        if st == 0:
            lib.mnnb200_exec_destroy(h)
        assert st == want, (blocks, st)
    st, h = create_linear(backend, 2048, oc, np.zeros(oc * 1024, np.uint8), np.ones((oc, 2), np.float32), bits=4)   # blocks of 1024
    if st == 0:
        lib.mnnb200_exec_destroy(h)
    assert st == nsup
    st, h = create_linear(backend, 511, oc, np.zeros(oc * 256, np.uint8), np.ones((oc, 1), np.float32), bits=4)   # odd ic
    if st == 0:
        lib.mnnb200_exec_destroy(h)
    assert st == nsup


@pytest.mark.gpu
def test_w4_lm_head_takes_half_the_device_memory(backend):
    """a 151936 x 2048 lm_head (Qwen's vocabulary): the 4-bit execution holds about half the bytes of the 8-bit one"""
    import torch
    from mnn_b200 import _capi
    lib = _capi.lib()
    oc, ic = 151936, 2048
    al = np.full((oc, 1), 0.01, np.float32)
    used = {}
    for bits in (8, 4):
        w = np.zeros(oc * ic // (2 if bits == 4 else 1), np.uint8 if bits == 4 else np.int8)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        st, h = create_linear(backend, ic, oc, w, al, bits=bits)
        _capi.check(st)
        backend.onSync()
        torch.cuda.synchronize()
        used[bits] = free0 - torch.cuda.mem_get_info()[0]
        lib.mnnb200_exec_destroy(h)
    ratio = used[4] / used[8]
    assert used[8] >= oc * ic and 0.45 <= ratio <= 0.55, f"8-bit {used[8]} bytes, 4-bit {used[4]} bytes ({ratio:.3f})"


@pytest.mark.gpu
def test_w4_linear_through_reference_executor_on_plugin():
    """every golden case through the reference's Executor on MNN_FORWARD_CUDA (the plugin): created there, nothing declined,
    within GOLDEN_TOL of the recorded reference; a 2048-wide layer in blocks of 64 (whose halved width of 1024 also splits into 32
    blocks, so a plugin that took ic from the packed weight size created it) equals the reference; a layer in blocks of 16
    channels, which the ABI refuses, is declined and runs on the CPU backup backend"""
    if not W.have_reference():
        pytest.skip("the reference core and its 4-bit harness (oracle/_ref) are not in this snapshot")
    if not os.path.exists(PLUGIN):
        pytest.fail("mnn_b200/libmnn_b200_plugin.so is missing although the reference core is present")
    for j, (x, wp, alpha, _, wmin, bias, gold) in enumerate(golden_cases(4)):
        y, stats, r = run_on_plugin(x, wp, alpha, wmin, bias, alpha.shape[1], 4)
        assert stats, r.stdout[-500:]
        assert stats["plugin_created"] >= 1 and stats["plugin_declined"] == 0, f"golden {j}: {stats}"
        assert np.abs(y - gold).max() <= GOLDEN_TOL * np.abs(gold).max(), f"golden {j}: {np.abs(y - gold).max() / np.abs(gold).max()}"
    rng = np.random.default_rng(2048)
    x, wp, alpha, wzero, bias = linear_data(rng, 4, 2048, 64, False, True, bits=4, bs=64)
    y, stats, r = run_on_plugin(x, wp, alpha, None, bias, 32, 4)
    assert stats and stats["plugin_created"] >= 1 and stats["plugin_declined"] == 0, f"{stats} {r.stdout[-800:]}"
    ref = W.linear_w4_dynamic_blocks(x, wp, 64, alpha, None, bias, 32)
    assert np.abs(y - ref).max() <= GOLDEN_TOL * np.abs(ref).max(), f"2048-wide 4-bit layer: {np.abs(y - ref).max() / np.abs(ref).max()}"
    x, wp, alpha, wzero, bias = linear_data(rng, 3, 256, 48, False, True, bits=4, bs=16)
    y, stats, r = run_on_plugin(x, wp, alpha, None, bias, 16, 4)
    assert stats and stats["plugin_declined"] >= 1, f"a 16-channel-block layer was not declined: {stats} {r.stdout[-500:]}"
    # the backup backend runs it in its own arithmetic (the CPU's), not through the plugin: close to the oracle, not equal
    ref = W.linear_w4_dynamic_blocks(x, wp, 48, alpha, None, bias, 16)
    assert np.abs(y - ref).max() <= 1e-2 * np.abs(ref).max(), f"declined layer: {np.abs(y - ref).max() / np.abs(ref).max()}"


if __name__ == "__main__":       # test_w4_linear_launches_listed_kernels' child
    profile_golden_cases(4)
