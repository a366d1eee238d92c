"""The LLM linear layer with K-blocked int8 weight scales (MNN-LLM's quant_block export) on the GPU (-m gpu):
mnnb200_linear_w8_create_blocked runs on the existing GEMM (>= 9 tokens) and GEMV (<= 8 tokens) kernel instantiations and must
equal O.linear_w8_dynamic_blocks bit for bit, NaN-poisoned outputs included; the GEMV and the GEMM agree bit for bit for 2..8
tokens.  The plugin cases drive the reference's own Executor through libmnn_b200_plugin.so (skipped without oracle/_ref)."""
import ctypes as C
import json
import os
import struct
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from oracle import oracle as O
from tests.test_gpu_dispatch import KERNEL_TESTS, WGMMA_KEY, expect, launched, ok

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "block_linear_golden.npz")
PLUGIN = os.path.join(ROOT, "mnn_b200", "libmnn_b200_plugin.so")


def status_codes():
    """(INVALID_VALUE, NOT_SUPPORT) as the header spells them"""
    import re
    h = open(os.path.join(ROOT, "include", "mnn_b200.h")).read()
    return tuple(int(re.search(rf"MNNB200_{n}\s*=\s*(-?\d+)", h).group(1)) for n in ("INVALID_VALUE", "NOT_SUPPORT"))


def golden_cases():
    g = np.load(GOLD)
    out = []
    for j in range(int(g["n"])):
        alpha, wmin, bias = g[f"b{j}_alpha"], g[f"b{j}_wmin"], g[f"b{j}_bias"]
        wz = (wmin - np.float32(-128) * alpha).astype(np.float32) if wmin.size else None
        out.append((g[f"b{j}_x"], g[f"b{j}_wq"], alpha, wz, wmin if wmin.size else None, bias if bias.size else None, g[f"b{j}_y"]))
    return out


def block_data(rng, tokens, ic, oc, bs, asym, has_bias):
    blocks = ic // bs
    x = rng.uniform(-1, 1, (tokens, ic)).astype(np.float32)
    wq = rng.integers(-128, 128, (oc, ic), dtype=np.int8)
    alpha = rng.uniform(0.001, 0.01, (oc, blocks)).astype(np.float32)
    wzero = rng.uniform(-0.05, 0.05, (oc, blocks)).astype(np.float32) if asym else None
    bias = rng.uniform(-1, 1, oc).astype(np.float32) if has_bias else None
    return x, wq, alpha, wzero, bias


def run_blocked(backend, x, wq, alpha, wzero, bias, variants, relu6=False, misalign=False, profile=False):
    """the layer at each variant (0 auto, 2 GEMM, 4 GEMV) on one execution, outputs NaN-poisoned first: {variant: (y, keys)}.
    profile: run each under torch.profiler (test_gpu_dispatch.launched) and return the launched kernel keys, else keys = None."""
    import torch
    from mnn_b200 import _capi
    from mnn_b200.backend import Op, Tensor
    tokens, ic = x.shape
    oc = wq.shape[0]
    op = Op(type="LinearW8", conv=dict(ic=ic, oc=oc, kernel=(1, 1)), weight=wq, wscale=alpha, wzero=wzero, bias=bias,
            relu6=relu6)
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


def variants_for(tokens):
    return (0,) if tokens == 1 else (0, 2, 4) if tokens <= 8 else (0, 2)


def check_blocked(backend, x, wq, alpha, wzero, bias, relu6=False, misalign=False, profile=False):
    """auto (and the forced GEMM / GEMV where they apply) against the oracle, bit for bit; returns the output.  profile: also
    every launched kernel is one of the instantiations KERNEL_TESTS lists (blocked layers add no entry point)"""
    tokens = x.shape[0]
    ref = O.linear_w8_dynamic_blocks(x, wq, alpha, wzero, bias, alpha.shape[1], relu6=relu6)
    res = run_blocked(backend, x, wq, alpha, wzero, bias, variants_for(tokens), relu6=relu6, misalign=misalign, profile=profile)
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
    for j, (x, wq, alpha, wz, _, bias, gold) in enumerate(golden_cases()):
        y = check_blocked(backend, x, wq, alpha, wz, bias, profile=profile)
        assert np.abs(y - gold).max() <= 4e-6 * np.abs(gold).max(), f"golden {j}: {np.abs(y - gold).max() / np.abs(gold).max()}"


@pytest.mark.gpu
def test_block_linear_golden_cases(backend):
    golden_check(backend, profile=False)


@pytest.mark.gpu
def test_block_linear_launches_listed_kernels():
    """the golden cases again, every variant under torch.profiler: only kernel instantiations KERNEL_TESTS lists are launched,
    the GEMM for the forced tensor-core variant, the GEMV alone for <= 8 tokens.  In a child process: a profiler that this
    module starts early in the GPU suite leaves CUPTI subscribed (test_gpu_dispatch keeps it so), and the windows
    test_gpu_dispatch opens later in the same process then recorded no kernel launches."""
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-m", "tests.test_gpu_block_linear"]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "golden cases profiled" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


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
    x, wq, alpha, wzero, bias = block_data(rng, tokens, ic, oc, bs, asym, has_bias)
    check_blocked(backend, x, wq, alpha, wzero, bias, relu6=relu6)


@pytest.mark.gpu
@pytest.mark.parametrize("tokens", [1, 3, 20])
def test_block_linear_relu_zero_row_misaligned(backend, tokens):
    """relu (conv flag), an all-zero token row (the amax < 1e-7 / range <= 1e-7 branches) and x 4 bytes past alignment"""
    import torch
    from mnn_b200 import _capi
    from mnn_b200.backend import Op, Tensor
    rng = np.random.default_rng(5 + tokens)
    x, wq, alpha, wzero, bias = block_data(rng, tokens, 1024, 72, 64, True, True)
    x[tokens // 2] = 0
    check_blocked(backend, x, wq, alpha, wzero, bias, misalign=True)
    ref = O.linear_w8_dynamic_blocks(x, wq, alpha, wzero, bias, alpha.shape[1], relu=True)
    op = Op(type="LinearW8", conv=dict(ic=1024, oc=72, kernel=(1, 1), relu=True), weight=wq, wscale=alpha, wzero=wzero, bias=bias)
    xin = Tensor((tokens, 1024), "float", data=torch.from_numpy(x).cuda())
    yout = Tensor((tokens, 72), "float")
    ex = backend.onCreate([xin], [yout], op)
    assert ex is not None and ex.onResize([xin], [yout]) == 0
    yout.data = torch.full((tokens, 72), float("nan"), dtype=torch.float32, device="cuda")
    _capi.check(ex.onExecute([xin], [yout]))
    backend.onSync()
    assert np.array_equal(yout.data.cpu().numpy(), ref)


def _create(backend, ic, oc, blocks, wq, alpha, wzero=None, bias=None):
    from mnn_b200 import _capi
    h = C.c_void_p()
    ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    st = _capi.lib().mnnb200_linear_w8_create_blocked(backend.runtime._h, ic, oc, blocks, ptr(wq), ptr(alpha), ptr(wzero),
                                                      ptr(bias), 0, 0, C.byref(h))
    return st, h


@pytest.mark.gpu
def test_block_linear_variants_and_validation(backend):
    import torch
    from mnn_b200 import _capi
    lib = _capi.lib()
    inval, nsup = status_codes()
    rng = np.random.default_rng(3)
    ic, oc = 512, 96
    for tokens in (2, 5, 8):        # GEMV (variant 4) and GEMM (variant 2): identical bits
        x, wq, alpha, wzero, bias = block_data(rng, tokens, ic, oc, 64, True, True)
        res = run_blocked(backend, x, wq, alpha, wzero, bias, (4, 2))
        assert np.array_equal(res[4][0], res[2][0]), f"{tokens} tokens: GEMV and GEMM differ"
    x, wq, alpha, wzero, bias = block_data(rng, 300, ic, oc, 64, True, True)
    st, h = _create(backend, ic, oc, ic // 64, wq, alpha, wzero, bias)
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
    # blocks == 1 through the blocked entry is the per-channel layer, bit for bit
    for tokens in (1, 4, 40):
        x, wq, alpha, wzero, bias = block_data(rng, tokens, ic, oc, ic, True, True)
        yb = run_blocked(backend, x, wq, alpha, wzero, bias, (0,))[0][0]
        yc = run_blocked(backend, x, wq, alpha[:, 0].copy(), wzero[:, 0].copy(), bias, (0,))[0][0]
        assert np.array_equal(yb, yc)
    wq = np.zeros((oc, ic), np.int8)
    for blocks, want in ((0, inval), (-1, inval), (3, inval), (ic // 16, nsup), (5, inval)):
        al = np.ones((oc, max(blocks, 1)), np.float32)
        st, h = _create(backend, ic, oc, blocks, wq, al)
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
    env = dict(os.environ, REFDUMP_PLUGIN=PLUGIN)
    env["LD_LIBRARY_PATH"] = O.REF_DIR + ":" + os.path.join(ROOT, "mnn_b200") + ":" + env.get("LD_LIBRARY_PATH", "")

    def run(x, wq, alpha, wmin, bias, blocks):
        tokens, ic = x.shape
        oc = wq.shape[0]
        al = np.stack([wmin, alpha], 2).astype(np.float32).ravel() if wmin is not None else alpha.astype(np.float32).ravel()
        payload = struct.pack("<8i", tokens, ic, oc, int(wmin is not None), 0, 0, int(bias is not None), blocks)
        payload += x.tobytes() + wq.tobytes() + al.tobytes() + (bias.astype(np.float32).tobytes() if bias is not None else b"")
        with tempfile.TemporaryDirectory() as d:
            req, out = os.path.join(d, "req.bin"), os.path.join(d, "out.bin")
            open(req, "wb").write(payload)
            r = subprocess.run([O.REFDUMP, "linear", req, out, "1"], env=env, capture_output=True, text=True, timeout=300)
            assert r.returncode == 0, r.stderr[-1500:]
            stats = [json.loads(l) for l in r.stdout.splitlines() if l.startswith("{\"plugin_")]
            return np.fromfile(out, np.float32).reshape(tokens, oc), (stats[-1] if stats else None), r

    for j, (x, wq, alpha, _, wmin, bias, gold) in enumerate(golden_cases()):
        y, stats, r = run(x, wq, alpha, wmin, bias, alpha.shape[1])
        assert stats, r.stdout[-500:]
        assert stats["plugin_created"] >= 1 and stats["plugin_declined"] == 0, f"golden {j}: {stats} {r.stderr[-800:]}"
        assert np.abs(y - gold).max() <= 4e-6 * np.abs(gold).max(), f"golden {j}: {np.abs(y - gold).max() / np.abs(gold).max()}"
    rng = np.random.default_rng(16)
    x, wq, alpha, wzero, bias = block_data(rng, 3, 256, 48, 16, False, True)
    y, stats, r = run(x, wq, alpha, None, bias, 16)
    assert stats and stats["plugin_declined"] >= 1, f"a 16-channel-block layer was not declined: {stats} {r.stdout[-500:]}"
    # the backup backend runs it in its own float arithmetic, not the W8A8 one of the oracle: close, not equal
    ref = O.linear_w8_dynamic_blocks(x, wq, alpha, None, bias, 16)
    assert np.abs(y - ref).max() <= 1e-2 * np.abs(ref).max(), f"declined layer: {np.abs(y - ref).max() / np.abs(ref).max()}"


if __name__ == "__main__":       # test_block_linear_launches_listed_kernels' child: the session backend of tests/conftest.py
    import torch
    from mnn_b200.backend import Runtime
    torch.cuda.set_stream(torch.cuda.Stream())
    golden_check(Runtime(0).onCreate(), profile=True)
    print("golden cases profiled")
