"""The LLM linear layer with 4-bit weights (MNN-LLM's default --quant_bit 4 export) on the GPU (-m gpu):
mnnb200_linear_w4_create_blocked keeps only the packed nibbles on the device and runs on the existing GEMM (>= 9 tokens, the
nibbles expanded in shared memory) and GEMV (<= 8 tokens, expanded in registers) kernel instantiations.  Every output must equal
W.linear_w4_dynamic_blocks bit for bit, NaN-poisoned outputs included; the GEMV and the GEMM agree bit for bit for 2..8 tokens.
The plugin cases drive the reference's own Executor through libmnn_b200_plugin.so (skipped without oracle/_ref)."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as O
from oracle import w4_oracle as W
from tests.test_gpu_block_linear import PLUGIN, ROOT, status_codes, variants_for
from tests.test_gpu_dispatch import KERNEL_TESTS, WGMMA_KEY, expect, launched, ok

GOLD = os.path.join(ROOT, "tests", "golden", "w4_linear_golden.npz")
TOL = 4e-6          # of max|y|: the oracle against the recorded reference (tests/test_w4_linear_cpu.py)


def golden_cases():
    g = np.load(GOLD)
    out = []
    for j in range(int(g["n"])):
        alpha, wmin, bias = g[f"c{j}_alpha"], g[f"c{j}_wmin"], g[f"c{j}_bias"]
        wz = (wmin - np.float32(-8) * alpha).astype(np.float32) if wmin.size else None      # what load() hands a backend
        out.append((g[f"c{j}_x"], g[f"c{j}_w"], alpha, wz, wmin if wmin.size else None, bias if bias.size else None, g[f"c{j}_y"]))
    return out


def w4_data(rng, tokens, ic, oc, bs, asym, has_bias):
    """bs 0: per channel.  Returns x, the packed weights, alpha / wzero [oc][blocks] (wzero as load() returns it), bias"""
    blocks = ic // bs if bs else 1
    x = rng.uniform(-1, 1, (tokens, ic)).astype(np.float32)
    wp = W.pack_w4(rng.integers(-8, 8, (oc, ic)))
    alpha = rng.uniform(0.001, 0.01, (oc, blocks)).astype(np.float32)
    wzero = rng.uniform(-0.01, 0.09, (oc, blocks)).astype(np.float32) if asym else None
    bias = rng.uniform(-1, 1, oc).astype(np.float32) if has_bias else None
    return x, wp, alpha, wzero, bias


def run_w4(backend, x, wp, alpha, wzero, bias, variants, relu=False, relu6=False, misalign=False, profile=False):
    """the layer at each variant (0 auto, 2 GEMM, 4 GEMV) on one execution created through Op(bits=4), outputs NaN-poisoned
    first: {variant: (y, keys)}; keys are the launched kernels under torch.profiler when profile is set"""
    import torch
    from mnn_b200 import _capi
    from mnn_b200.backend import Op, Tensor
    tokens, ic = x.shape
    oc = alpha.shape[0]
    al = alpha if alpha.shape[1] > 1 else alpha[:, 0].copy()
    wz = None if wzero is None else (wzero if wzero.shape[1] > 1 else wzero[:, 0].copy())
    op = Op(type="LinearW8", conv=dict(ic=ic, oc=oc, kernel=(1, 1), relu=relu), weight=wp, wscale=al, wzero=wz, bias=bias,
            relu6=relu6, bits=4)
    if misalign:        # a view 4 bytes into a buffer: x is 4 bytes past 16-byte alignment
        buf = torch.zeros(tokens * ic + 8, dtype=torch.float32, device="cuda")
        xd = buf[1:1 + tokens * ic].view(tokens, ic)
        xd.copy_(torch.from_numpy(x))
        assert xd.data_ptr() % 16 == 4
    else:
        xd = torch.from_numpy(x).cuda()
    xin = Tensor((tokens, ic), "float", data=xd)
    yout = Tensor((tokens, oc), "float")
    ex = backend.onCreate([xin], [yout], op)
    assert ex is not None and ex.onResize([xin], [yout]) == 0
    yout.data = torch.empty((tokens, oc), dtype=torch.float32, device="cuda")
    res = {}
    for v in variants:
        _capi.check(_capi.lib().mnnb200_conv_int8_set_variant(ex._h, v))
        keys = None
        if profile:
            keys = launched(backend, lambda: ok(ex.onExecute([xin], [yout])), lambda: yout.data.fill_(float("nan")))
        else:
            yout.data.fill_(float("nan"))
            ok(ex.onExecute([xin], [yout]))
            backend.onSync()
        y = yout.data.cpu().numpy()
        assert not np.isnan(y).any(), f"variant {v}: outputs left unwritten"
        res[v] = (y, keys)
    return res


def check_w4(backend, x, wp, alpha, wzero, bias, relu=False, relu6=False, misalign=False, profile=False):
    """auto (and the forced GEMM / GEMV where they apply) against the oracle, bit for bit; returns the oracle's output"""
    tokens = x.shape[0]
    ref = W.linear_w4_dynamic_blocks(x, wp, alpha.shape[0], alpha, wzero, bias, alpha.shape[1], relu=relu, relu6=relu6)
    res = run_w4(backend, x, wp, alpha, wzero, bias, variants_for(tokens), relu=relu, relu6=relu6, misalign=misalign,
                 profile=profile)
    for v, (y, keys) in res.items():
        assert np.array_equal(y, ref), f"variant {v}: {np.count_nonzero(y != ref)} outputs differ, max {np.abs(y - ref).max()}"
        if profile:
            assert set(keys) <= set(KERNEL_TESTS), f"variant {v} launched kernels outside KERNEL_TESTS: {sorted(keys)}"
            if v == 2 or (v == 0 and tokens > 8):
                expect(keys, WGMMA_KEY)
            if v == 4 or (v == 0 and tokens <= 8):
                assert {k[0] for k in keys} == {"linear_w8_gemv_kernel"}, sorted(keys)
    return ref


def golden_check(backend, profile):
    for j, (x, wp, alpha, wz, _, bias, gold) in enumerate(golden_cases()):
        y = check_w4(backend, x, wp, alpha, wz, bias, profile=profile)
        assert np.abs(y - gold).max() <= TOL * np.abs(gold).max(), f"golden {j}: {np.abs(y - gold).max() / np.abs(gold).max()}"


@pytest.mark.gpu
def test_w4_linear_golden_cases(backend):
    golden_check(backend, profile=False)


@pytest.mark.gpu
def test_w4_linear_launches_listed_kernels():
    """the golden cases again, every variant under torch.profiler: only instantiations KERNEL_TESTS lists are launched (in a
    child process, for the reason test_block_linear_launches_listed_kernels gives)"""
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-m", "tests.test_gpu_w4_linear"]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "golden cases profiled" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


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
    x, wp, alpha, wzero, bias = w4_data(rng, tokens, ic, oc, bs, asym, has_bias)
    check_w4(backend, x, wp, alpha, wzero, bias, relu=relu, relu6=relu6)


@pytest.mark.gpu
@pytest.mark.parametrize("tokens,bs", [(1, 64), (3, 0), (20, 64), (300, 128)])
def test_w4_linear_zero_row_misaligned(backend, tokens, bs):
    """an all-zero token row (the amax < 1e-7 / range <= 1e-7 branches) and x 4 bytes past 16-byte alignment"""
    rng = np.random.default_rng(5 + tokens)
    x, wp, alpha, wzero, bias = w4_data(rng, tokens, 1024, 72, bs, True, True)
    x[tokens // 2] = 0
    check_w4(backend, x, wp, alpha, wzero, bias, misalign=True)


def _create(backend, ic, oc, blocks, wp, alpha, wzero=None, bias=None):
    from mnn_b200 import _capi
    h = C.c_void_p()
    ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    st = _capi.lib().mnnb200_linear_w4_create_blocked(backend.runtime._h, ic, oc, blocks, ptr(wp), ptr(alpha), ptr(wzero),
                                                      ptr(bias), 0, 0, C.byref(h))
    return st, h


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
            x, wp, alpha, wzero, bias = w4_data(rng, tokens, ic, oc, bs, True, True)
            res = run_w4(backend, x, wp, alpha, wzero, bias, (4, 2))
            assert np.array_equal(res[4][0], res[2][0]), f"{tokens} tokens, bs {bs}: GEMV and GEMM differ"
    x, wp, alpha, wzero, bias = w4_data(rng, 300, ic, oc, 64, True, True)
    st, h = _create(backend, ic, oc, ic // 64, wp, alpha, wzero, bias)
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
        st, h = _create(backend, ic, oc, blocks, wp, al)
        if st == 0:
            lib.mnnb200_exec_destroy(h)
        assert st == want, (blocks, st)
    st, h = _create(backend, 2048, oc, 2, np.zeros(oc * 1024, np.uint8), np.ones((oc, 2), np.float32))   # blocks of 1024
    if st == 0:
        lib.mnnb200_exec_destroy(h)
    assert st == nsup
    st, h = _create(backend, 511, oc, 1, np.zeros(oc * 256, np.uint8), np.ones(oc, np.float32))          # odd ic
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
    al = np.full(oc, 0.01, np.float32)
    used = {}
    for bits in (8, 4):
        w = np.zeros(oc * ic // (2 if bits == 4 else 1), np.uint8 if bits == 4 else np.int8)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        h = C.c_void_p()
        fn = lib.mnnb200_linear_w4_create_blocked if bits == 4 else lib.mnnb200_linear_w8_create_blocked
        _capi.check(fn(backend.runtime._h, ic, oc, 1, w.ctypes.data_as(C.c_void_p), al.ctypes.data_as(C.c_void_p), None, None,
                       0, 0, C.byref(h)))
        backend.onSync()
        torch.cuda.synchronize()
        used[bits] = free0 - torch.cuda.mem_get_info()[0]
        lib.mnnb200_exec_destroy(h)
    ratio = used[4] / used[8]
    assert used[8] >= oc * ic and 0.45 <= ratio <= 0.55, f"8-bit {used[8]} bytes, 4-bit {used[4]} bytes ({ratio:.3f})"


@pytest.mark.gpu
def test_w4_linear_through_reference_executor_on_plugin():
    """every golden case through the reference's Executor on MNN_FORWARD_CUDA (the plugin): created there, nothing declined,
    within TOL of the recorded reference; a 2048-wide layer in blocks of 64 (whose halved width of 1024 also splits into 32
    blocks, so a plugin that took ic from the packed weight size created it) equals the reference; a layer in blocks of 16
    channels, which the ABI refuses, is declined and runs on the CPU backup backend"""
    if not W.have_reference():
        pytest.skip("the reference core and its 4-bit harness (oracle/_ref) are not in this snapshot")
    if not os.path.exists(PLUGIN):
        pytest.fail("mnn_b200/libmnn_b200_plugin.so is missing although the reference core is present")
    env = dict(os.environ, REFDUMP_PLUGIN=PLUGIN)
    env["LD_LIBRARY_PATH"] = O.REF_DIR + ":" + os.path.join(ROOT, "mnn_b200") + ":" + env.get("LD_LIBRARY_PATH", "")

    def run(x, wp, alpha, wmin, bias, blocks):
        oc = alpha.shape[0]
        al = np.stack([wmin, alpha], 2).ravel() if wmin is not None else alpha.ravel()
        payload = W.linear_request(x, W.unpack_w4(wp, oc), al, wmin is not None, bias, blocks)
        y, out = W.run_refdump(payload, x.shape[0], oc, env=env)
        stats = [json.loads(l) for l in out.splitlines() if l.startswith("{\"plugin_")]
        return y, (stats[-1] if stats else None), out

    for j, (x, wp, alpha, _, wmin, bias, gold) in enumerate(golden_cases()):
        y, stats, r = run(x, wp, alpha, wmin, bias, alpha.shape[1])
        assert stats, r[-500:]
        assert stats["plugin_created"] >= 1 and stats["plugin_declined"] == 0, f"golden {j}: {stats}"
        assert np.abs(y - gold).max() <= TOL * np.abs(gold).max(), f"golden {j}: {np.abs(y - gold).max() / np.abs(gold).max()}"
    rng = np.random.default_rng(2048)
    x, wp, alpha, wzero, bias = w4_data(rng, 4, 2048, 64, 64, False, True)
    y, stats, r = run(x, wp, alpha, None, bias, 32)
    assert stats and stats["plugin_created"] >= 1 and stats["plugin_declined"] == 0, f"{stats} {r[-800:]}"
    ref = W.linear_w4_dynamic_blocks(x, wp, 64, alpha, None, bias, 32)
    assert np.abs(y - ref).max() <= TOL * np.abs(ref).max(), f"2048-wide 4-bit layer: {np.abs(y - ref).max() / np.abs(ref).max()}"
    x, wp, alpha, wzero, bias = w4_data(rng, 3, 256, 48, 16, False, True)
    y, stats, r = run(x, wp, alpha, None, bias, 16)
    assert stats and stats["plugin_declined"] >= 1, f"a 16-channel-block layer was not declined: {stats} {r[-500:]}"
    # the backup backend runs it in its own arithmetic (the CPU's), not through the plugin: close to the oracle, not equal
    ref = W.linear_w4_dynamic_blocks(x, wp, 48, alpha, None, bias, 16)
    assert np.abs(y - ref).max() <= 1e-2 * np.abs(ref).max(), f"declined layer: {np.abs(y - ref).max() / np.abs(ref).max()}"


if __name__ == "__main__":       # test_w4_linear_launches_listed_kernels' child: the session backend of tests/conftest.py
    import torch
    from mnn_b200.backend import Runtime
    torch.cuda.set_stream(torch.cuda.Stream())
    golden_check(Runtime(0).onCreate(), profile=True)
    print("golden cases profiled")
