"""The LLM linear layer with K-blocked int8 weight scales (MNN-LLM's quant_block export) on the GPU (-m gpu):
mnnb200_linear_w8_create_blocked runs on the existing GEMM (>= 9 tokens) and GEMV (<= 8 tokens) kernel instantiations and must
equal O.linear_w8_dynamic_blocks bit for bit, NaN-poisoned outputs included; the GEMV and the GEMM agree bit for bit for 2..8
tokens.  The plugin cases drive the reference's own Executor through libmnn_b200_plugin.so (skipped without oracle/_ref)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
from oracle import w4_oracle as W
from tests.test_gpu_dispatch import (ROOT, check_linear, create_linear, golden_cases, golden_check, golden_check_profiled_in_child,
                                     linear_data, profile_golden_cases, run_linear)

PLUGIN = os.path.join(ROOT, "mnn_b200", "libmnn_b200_plugin.so")


def status_codes():
    """(INVALID_VALUE, NOT_SUPPORT) as the header spells them"""
    import re
    h = open(os.path.join(ROOT, "include", "mnn_b200.h")).read()
    return tuple(int(re.search(rf"MNNB200_{n}\s*=\s*(-?\d+)", h).group(1)) for n in ("INVALID_VALUE", "NOT_SUPPORT"))


def run_on_plugin(x, w, alpha, wmin, bias, blocks, bits=8):
    """one linear layer (wmin: the wire min or None) through the reference's Executor on MNN_FORWARD_CUDA, the plugin loaded
    into refdump (4-bit: refdump_w4): (y, the plugin's last stats line or None, the finished process)"""
    env = dict(os.environ, REFDUMP_PLUGIN=PLUGIN)
    env["LD_LIBRARY_PATH"] = O.REF_DIR + ":" + os.path.join(ROOT, "mnn_b200") + ":" + env.get("LD_LIBRARY_PATH", "")
    oc = alpha.shape[0]
    q = W.unpack_w4(w, oc) if bits == 4 else w
    al = np.stack([wmin, alpha], 2) if wmin is not None else alpha         # {min, scale} pairs when asymmetric
    payload = O.linear_request(x, q, al.ravel(), wmin is not None, bias, blocks)
    y, r = O.run_linear_request(payload, x.shape[0], oc, W.REFDUMP_W4 if bits == 4 else O.REFDUMP, env=env)
    stats = [json.loads(l) for l in r.stdout.splitlines() if l.startswith("{\"plugin_")]
    return y, (stats[-1] if stats else None), r


@pytest.mark.gpu
def test_block_linear_golden_cases(backend):
    golden_check(backend, 8)


@pytest.mark.gpu
def test_block_linear_launches_listed_kernels():
    """the golden cases again, every variant under torch.profiler: only kernel instantiations KERNEL_TESTS lists are launched,
    the GEMM for the forced tensor-core variant, the GEMV alone for <= 8 tokens.  In a child process: a profiler that this
    module starts early in the GPU suite leaves CUPTI subscribed (test_gpu_dispatch keeps it so), and the windows
    test_gpu_dispatch opens later in the same process then recorded no kernel launches."""
    golden_check_profiled_in_child("tests.test_gpu_block_linear")


SWEEP = [  # (tokens, ic, oc, bs, asym, bias, relu6)
    (1, 256, 40, 32, True, True, False), (1, 5504, 264, 64, True, True, False), (1, 2048, 33, 128, False, False, True),
    (1, 1024, 300, 256, True, False, False), (1, 1024, 16, 512, True, True, False),
    (2, 2048, 2100, 64, True, True, False), (2, 512, 33, 32, False, True, False), (5, 5504, 48, 64, True, False, True),
    (5, 768, 40, 256, False, False, False), (8, 1024, 520, 128, True, True, False), (8, 2048, 4300, 64, False, True, False),
    (9, 256, 33, 32, True, True, False), (9, 5504, 200, 64, True, True, False), (100, 2048, 2048, 128, True, False, False),
    (100, 1024, 40, 256, False, True, True), (256, 5504, 600, 64, True, True, False), (256, 640, 1000, 32, True, True, False),
    (300, 2048, 528, 64, False, False, False), (300, 1536, 2056, 128, True, True, False), (512, 2048, 2048, 64, True, True, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("tokens,ic,oc,bs,asym,has_bias,relu6", SWEEP)
def test_block_linear_sweep(backend, tokens, ic, oc, bs, asym, has_bias, relu6):
    rng = np.random.default_rng(tokens * 7919 + ic * 31 + oc + bs)
    x, wq, alpha, wzero, bias = linear_data(rng, tokens, ic, oc, asym, has_bias, bs=bs)
    check_linear(backend, x, wq, alpha, wzero, bias, relu6=relu6)


@pytest.mark.gpu
@pytest.mark.parametrize("tokens", [1, 3, 20])
def test_block_linear_relu_zero_row_misaligned(backend, tokens):
    """relu (conv flag), an all-zero token row (the amax < 1e-7 / range <= 1e-7 branches) and x 4 bytes past alignment"""
    rng = np.random.default_rng(5 + tokens)
    x, wq, alpha, wzero, bias = linear_data(rng, tokens, 1024, 72, True, True, bs=64)
    x[tokens // 2] = 0
    check_linear(backend, x, wq, alpha, wzero, bias, misalign=True)
    ref = O.linear_w8_dynamic_blocks(x, wq, alpha, wzero, bias, alpha.shape[1], relu=True)
    y = run_linear(backend, x, wq, alpha, wzero, bias, (0,), relu=True)[0][0]
    assert np.array_equal(y, ref)


@pytest.mark.gpu
def test_block_linear_variants_and_validation(backend):
    import torch
    from mnn_b200 import _capi
    lib = _capi.lib()
    inval, nsup = status_codes()
    rng = np.random.default_rng(3)
    ic, oc = 512, 96
    for tokens in (2, 5, 8):        # GEMV (variant 4) and GEMM (variant 2): identical bits
        x, wq, alpha, wzero, bias = linear_data(rng, tokens, ic, oc, True, True, bs=64)
        res = run_linear(backend, x, wq, alpha, wzero, bias, (4, 2))
        assert np.array_equal(res[4][0], res[2][0]), f"{tokens} tokens: GEMV and GEMM differ"
    x, wq, alpha, wzero, bias = linear_data(rng, 300, ic, oc, True, True, bs=64)
    st, h = create_linear(backend, ic, oc, wq, alpha, wzero, bias)
    assert st == 0
    try:
        xd = torch.from_numpy(x).cuda()
        yd = torch.empty((300, oc), dtype=torch.float32, device="cuda")
        assert lib.mnnb200_linear_w8_resize(h, 300) == 0
        assert lib.mnnb200_conv_int8_set_variant(h, 3) == 0
        assert lib.mnnb200_linear_w8_execute(h, C.c_void_p(xd.data_ptr()), C.c_void_p(yd.data_ptr())) == nsup
        assert lib.mnnb200_linear_w8_resize(h, 1) == 0
        assert lib.mnnb200_conv_int8_set_variant(h, 2) == 0
        assert lib.mnnb200_linear_w8_execute(h, C.c_void_p(xd.data_ptr()), C.c_void_p(yd.data_ptr())) == nsup
    finally:
        lib.mnnb200_exec_destroy(h)
    # blocks == 1 through the blocked entry (the layer's Op) is the per-channel layer (mnnb200_linear_w8_create), bit for bit
    for tokens in (1, 4, 40):
        x, wq, alpha, wzero, bias = linear_data(rng, tokens, ic, oc, True, True, bs=ic)
        yb = run_linear(backend, x, wq, alpha, wzero, bias, (0,))[0][0]
        st, h = create_linear(backend, ic, oc, wq, alpha[:, 0].copy(), wzero[:, 0].copy(), bias)
        assert st == 0
        try:
            xd = torch.from_numpy(x).cuda()
            yd = torch.full((tokens, oc), float("nan"), dtype=torch.float32, device="cuda")
            assert lib.mnnb200_linear_w8_resize(h, tokens) == 0
            assert lib.mnnb200_linear_w8_execute(h, C.c_void_p(xd.data_ptr()), C.c_void_p(yd.data_ptr())) == 0
            backend.onSync()
        finally:
            lib.mnnb200_exec_destroy(h)
        assert np.array_equal(yb, yd.cpu().numpy())
    wq = np.zeros((oc, ic), np.int8)
    for blocks, want in ((0, inval), (-1, inval), (3, inval), (ic // 16, nsup), (5, inval)):
        al = np.ones((oc, max(blocks, 1)), np.float32)
        st, h = create_linear(backend, ic, oc, wq, al, blocks=blocks)
        if st == 0:
            lib.mnnb200_exec_destroy(h)
        assert st == want, (blocks, st)


@pytest.mark.gpu
def test_block_linear_through_reference_executor_on_plugin():
    """every golden case through the reference's Executor on MNN_FORWARD_CUDA (the plugin): created there, nothing declined,
    within 4e-6 of the recorded reference; a layer of 16-channel blocks is declined and runs on the CPU backup backend"""
    if not O.have_reference():
        pytest.skip("the reference core (oracle/_ref) is not in this snapshot")
    if not os.path.exists(PLUGIN):
        pytest.fail("mnn_b200/libmnn_b200_plugin.so is missing although the reference core is present")
    for j, (x, wq, alpha, _, wmin, bias, gold) in enumerate(golden_cases(8)):
        y, stats, r = run_on_plugin(x, wq, alpha, wmin, bias, alpha.shape[1])
        assert stats, r.stdout[-500:]
        assert stats["plugin_created"] >= 1 and stats["plugin_declined"] == 0, f"golden {j}: {stats} {r.stderr[-800:]}"
        assert np.abs(y - gold).max() <= 4e-6 * np.abs(gold).max(), f"golden {j}: {np.abs(y - gold).max() / np.abs(gold).max()}"
    rng = np.random.default_rng(16)
    x, wq, alpha, wzero, bias = linear_data(rng, 3, 256, 48, False, True, bs=16)
    y, stats, r = run_on_plugin(x, wq, alpha, None, bias, 16)
    assert stats and stats["plugin_declined"] >= 1, f"a 16-channel-block layer was not declined: {stats} {r.stdout[-500:]}"
    # the backup backend runs it in its own float arithmetic, not the W8A8 one of the oracle: close, not equal
    ref = O.linear_w8_dynamic_blocks(x, wq, alpha, None, bias, 16)
    assert np.abs(y - ref).max() <= 1e-2 * np.abs(ref).max(), f"declined layer: {np.abs(y - ref).max() / np.abs(ref).max()}"


if __name__ == "__main__":       # test_block_linear_launches_listed_kernels' child
    profile_golden_cases(8)
