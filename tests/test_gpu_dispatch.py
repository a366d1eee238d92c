"""One reference-checked case group per run-time dispatch branch of the int8 / linear kernels (-m gpu), and a CPU check that
every kernel entry point of the built library is named in KERNEL_TESTS with the test that launches it.

The launchers pick a template instantiation from the shape and the SM count: the GEMV's tokens and rows per warp
(linear_w8_gemv.cu: launch_r), the dynamic quantisation's vector width (elementwise.cu: launch_dynamic_quant), the mma.sync
tile (capi.cu: pick_tile), the stem's output-channel width (conv_int8_stem.cu) and the depthwise strip / generic kernel
(elementwise.cu: launch_dwconv_int8).  Every case below derives its shape from the SM count with the launcher's own rule,
runs under torch.profiler and asserts that the intended instantiation ran, so a case that dispatch moves off its branch fails
instead of silently losing coverage.  int8 outputs are poisoned before the run and must equal the oracle bit for bit with
zero NHWC16 channel padding; linear outputs are NaN-poisoned and must equal O.linear_w8_dynamic bit for bit and, for 2..8
tokens, the tensor-core path (variant 2)."""
import os
import re
import shutil
import subprocess
from collections import Counter

import numpy as np
import pytest

from oracle import oracle as O
from tests.cases import random_modern_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# torch.profiler (kineto) otherwise tears CUPTI down on a background thread after every profiling session, while this module
# opens one short session per case: keep CUPTI subscribed between them
os.environ.setdefault("TEARDOWN_CUPTI", "0")

# ---- every kernel entry point of libmnn_b200.so -> the test that launches it --------------------------------------------
# key: (base name, template arguments); bool arguments as 0 / 1, type arguments as spelled.  tools/kernel_coverage.py runs the
# GPU suite under torch.profiler and lists the launches of each entry, the evidence for the entries outside this module.
HERE = "tests/test_gpu_dispatch.py"
KERNEL_TESTS = {
    # decode GEMV: (tokens template, rows per warp, K chunks in flight)
    **{("linear_w8_gemv_kernel", (t, r, 4)): f"{HERE}::test_gemv_dispatch" for t in (1, 2, 4, 8) for r in (1, 2)},
    ("linear_w8_gemv_kernel", (1, 4, 4)): f"{HERE}::test_gemv_dispatch",
    ("linear_w8_gemv_kernel", (2, 4, 4)): f"{HERE}::test_gemv_dispatch",
    # prefill: per-token quantisation, then the tensor-core GEMM
    ("dynamic_quant_kernel", ()): f"{HERE}::test_prefill_dynamic_quant",
    ("dynamic_quant_vec_kernel", (2,)): f"{HERE}::test_prefill_dynamic_quant",
    ("dynamic_quant_vec_kernel", (4,)): f"{HERE}::test_prefill_dynamic_quant",
    ("dynamic_quant_vec_kernel", (8,)): f"{HERE}::test_prefill_dynamic_quant",
    ("gemm_i8_wgmma_kernel", (1, 0, 256)): f"{HERE}::test_prefill_dynamic_quant",
    ("gemm_i8_wgmma_kernel", (1, 1, 256)): "tests/test_gpu_parity.py::test_linear_w8_cta_pair_variant_bit_exact",
    ("gemm_i8_wgmma_kernel", (2, 0, 256)): "tests/test_gpu_winograd.py::test_wino_cell_matrix",
    # mma.sync implicit GEMM: (BM, BN, WM, WN)
    **{("conv_int8_igemm_kernel", t): f"{HERE}::test_mma_sync_tiles"
       for t in ((128, 64, 4, 2), (128, 32, 8, 1), (128, 16, 8, 1), (64, 64, 2, 2), (64, 32, 4, 1), (128, 128, 4, 2))},
    **{("conv_int8_stem_kernel", (ocp,)): f"{HERE}::test_stem" for ocp in (16, 32, 64)},
    ("dwconv3x3_int8_kernel", (1,)): f"{HERE}::test_depthwise_strip",
    ("dwconv3x3_int8_kernel", (2,)): f"{HERE}::test_depthwise_strip",
    ("dwconv_int8_kernel", ()): f"{HERE}::test_depthwise_generic",
    # the conv-group kernel, Winograd, fp32 conv / GEMM and the elementwise kernels: their own modules (the Winograd cell matrix
    # also runs every cell as three kernels, F(2,3)'s output transform only reachable that way)
    ("conv_group_wgmma_kernel", ()): "tests/test_gpu_conv_group.py::test_conv_group_width_by_chunk_matrix",
    ("wino_input_kernel", (4, 4)): "tests/test_gpu_winograd.py::test_wino_cell_matrix",
    ("wino_input_kernel", (8, 1)): "tests/test_gpu_winograd.py::test_wino_cell_matrix",
    ("wino_input_seq4_kernel", (6,)): "tests/test_gpu_winograd.py::test_wino_cell_matrix",
    ("wino_output_kernel", (4, 4)): "tests/test_gpu_winograd.py::test_wino_cell_matrix",
    ("wino_output_kernel", (6, 2)): "tests/test_gpu_winograd.py::test_wino_cell_matrix",
    ("wino_output_kernel", (8, 1)): "tests/test_gpu_winograd.py::test_wino_cell_matrix",
    ("wino_f23_fused_kernel", ()): "tests/test_gpu_winograd.py::test_wino_cell_matrix",
    ("conv_f32_wgmma_kernel", (32,)): "tests/test_gpu_conv_f32.py::test_conv_f32_cell_matrix",
    ("conv_f32_wgmma_kernel", (64,)): "tests/test_gpu_conv_f32.py::test_conv_f32_cell_matrix",
    ("conv_f32_wgmma_kernel", (128,)): "tests/test_gpu_conv_f32.py::test_conv_f32_cell_matrix",
    ("pack_conv_w_f32_kernel", ()): "tests/test_gpu_conv_f32.py::test_conv_f32_matches_float64",
    ("dwconv_f32_kernel", ()): "tests/test_gpu_conv_f32.py::test_dwconv_f32_matches_float64",
    ("scale_f32_kernel", ()): "tests/test_gpu_conv_f32.py::test_scale_f32",
    ("softmax_f32_kernel", ()): "tests/test_gpu_conv_f32.py::test_softmax_f32",
    ("gemm_f16_wgmma_kernel", (0,)): "tests/test_matmul.py::test_gpu_matmul_vs_float64",
    ("gemm_f16_wgmma_kernel", (1,)): "tests/test_matmul.py::test_gpu_matmul_vs_float64",
    ("pack_kmajor_f16_kernel", ("__half",)): "tests/test_matmul.py::test_gpu_matmul_vs_float64",
    ("pack_kmajor_f32_kernel", ("float",)): "tests/test_matmul.py::test_gpu_matmul_vs_float64",
    **{("binary_f32_kernel", (op,)): "tests/test_gpu_float_elementwise.py::test_binary_f32_bit_exact"
       for op in (0, 1, 2, 7, 8, 9, 14)},
    **{("unary_f32_kernel", (op,)): "tests/test_gpu_float_elementwise.py::test_unary_f32"
       for op in (0, 1, 4, 5, 6, 7, 8, 15, 29, 30, 31, 32, 33, 34)},
    ("argmax_f32_kernel", ()): "tests/test_gpu_float_elementwise.py::test_argmax_f32",
    ("float_to_int8_kernel", ()): "tests/test_gpu_parity.py::test_casts_vs_oracle",
    ("int8_to_float_kernel", ()): "tests/test_gpu_parity.py::test_casts_vs_oracle",
    ("pack_nchw_int8_kernel", ()): "tests/test_gpu_parity.py::test_casts_vs_oracle",
    ("unpack_nchw_int8_kernel", ()): "tests/test_gpu_parity.py::test_casts_vs_oracle",
    ("scale_int8_kernel", ()): "tests/test_gpu_parity.py::test_scale_and_pool_int8_vs_oracle",
    ("pool_int8_x86_kernel", ()): "tests/test_gpu_parity.py::test_scale_and_pool_int8_vs_oracle",
    ("binary_add_int8_kernel", ()): "tests/test_gpu_neighbours.py::test_add_int8_vs_oracle",
    ("avgpool_int8_via_float_kernel", ()): "tests/test_gpu_neighbours.py::test_avgpool_int8_vs_oracle",
    ("avgpool_int8_via_float_1ch_kernel", ()): "tests/test_gpu_neighbours.py::test_avgpool_int8_mobilenet_global",
    ("softmax_int8_kernel", ()): "tests/test_gpu_neighbours.py::test_softmax_int8",
    ("pool_f32_kernel", ()): "tests/test_gpu_neighbours.py::test_pool_f32_vs_oracle",
    ("relu_f32_kernel", ()): "tests/test_gpu_neighbours.py::test_relu_f32",
    ("reduce_f32_kernel", ()): "tests/test_gpu_neighbours.py::test_reduce_f32",
    ("raster_b32_kernel", ()): "tests/test_gpu_neighbours.py::test_raster_b32",
    ("transpose_b32_kernel", ()): "tests/test_gpu_neighbours.py::test_transpose_b32",
}


def _template_arg(a):
    a = re.sub(r"^\([A-Za-z_][\w: ]*\)", "", a.strip()).strip()     # cu++filt spells "(int)1", "(bool)0"; the profiler "1", "false"
    if a in ("true", "false"):
        return int(a == "true")
    return int(a) if re.fullmatch(r"-?\d+", a) else a


def kernel_key(name):
    """(base name, template arguments) of a demangled kernel name, as cu++filt or the CUDA profiler prints it"""
    s = name.replace("(anonymous namespace)", "anon").replace("<unnamed>", "anon").strip()
    if s.startswith("void "):
        s = s[5:]
    depth, end = 0, len(s)
    for i, ch in enumerate(s):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            end = i
            break
    head, args = s[:end].strip(), ()
    if head.endswith(">"):
        j = head.index("<")
        parts, depth, cur = [], 0, ""
        for ch in head[j + 1:-1]:
            if ch in "<(":
                depth += 1
            elif ch in ">)":
                depth -= 1
            if ch == "," and depth == 0:
                parts.append(cur)
                cur = ""
            else:
                cur += ch
        args = tuple(_template_arg(p) for p in parts + [cur])
        head = head[:j]
    return head.split("::")[-1], args


def _cuda_tool(name):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    path = os.path.join(os.path.dirname(nvcc), name)
    return path if os.path.exists(path) else shutil.which(name)


def library_kernels(lib_path):
    """kernel keys of every STO_ENTRY symbol of a built library"""
    cuobjdump, cufilt = _cuda_tool("cuobjdump"), _cuda_tool("cu++filt")
    assert cuobjdump and cufilt, "cuobjdump / cu++filt not found (CUDA toolkit)"
    out = subprocess.run([cuobjdump, "-symbols", lib_path], capture_output=True, text=True, check=True).stdout
    mangled = sorted({line.split()[-1] for line in out.splitlines() if "STO_ENTRY" in line})
    demangled = subprocess.run([cufilt], input="\n".join(mangled) + "\n", capture_output=True, text=True, check=True).stdout
    names = [d for d in demangled.splitlines() if d.strip()]
    assert len(names) == len(mangled) and mangled
    keys = [kernel_key(n) for n in names]
    assert len(set(keys)) == len(keys), "two entry points share one key: " + str(Counter(keys).most_common(3))
    return set(keys)


# ---- CPU: the table against the library ---------------------------------------------------------------------------------
def test_kernel_table_matches_library():
    from mnn_b200 import build as B
    lib = B.build()
    entries = library_kernels(lib)
    untested = sorted(entries - set(KERNEL_TESTS))
    stale = sorted(set(KERNEL_TESTS) - entries)
    assert not untested, f"kernel entry points with no test named in KERNEL_TESTS: {untested}"
    assert not stale, f"KERNEL_TESTS names kernels the library does not have: {stale}"


def test_kernel_table_names_existing_tests():
    for key, node in KERNEL_TESTS.items():
        path, func = node.split("::")
        with open(os.path.join(ROOT, path)) as f:
            assert re.search(rf"^def {func}\(", f.read(), re.M), f"{key}: {node} does not exist"


def test_kernel_name_formats_parse_alike():
    cufilt = "void mnnb200::<unnamed>::gemm_i8_wgmma_kernel<(int)1, (bool)0, (int)256>(CUtensorMap_st, CUtensorMap_st, mnnb200::<unnamed>::KParams)"
    prof = "void mnnb200::(anonymous namespace)::gemm_i8_wgmma_kernel<1, false, 256>(CUtensorMap_st, CUtensorMap_st, mnnb200::(anonymous namespace)::KParams)"
    assert kernel_key(cufilt) == kernel_key(prof) == ("gemm_i8_wgmma_kernel", (1, 0, 256))
    assert kernel_key("mnnb200::dwconv_int8_kernel(mnnb200::DwParams)") == ("dwconv_int8_kernel", ())
    assert kernel_key("void mnnb200::<unnamed>::pack_kmajor_f16_kernel<__half>(const T1 *, __half *, int, int, int, int)") == \
        ("pack_kmajor_f16_kernel", ("__half",))
    assert kernel_key("void mnnb200::binary_f32_kernel<(int)14>(const float *, const float *, float *, unsigned long, int, int, int, int)") == \
        kernel_key("void mnnb200::binary_f32_kernel<14>(float const*, float const*, float*, unsigned long, int, int, int, int)")


# ---- GPU helpers --------------------------------------------------------------------------------------------------------
LAUNCHED = Counter()        # every kernel key the cases of this module launched (read by tools/kernel_coverage.py)


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def launched(backend, fn, prepare):
    """prepare() (poison the output), then fn() under torch.profiler (CUDA activity): the kernel keys fn launched.
    A kernel's activity record reaches the profiler asynchronously, and now and then a window this short closes before it
    does (seen on the H100 in about one window in fifty, the kernel having run; such a window held an "Activity Buffer Request"
    after the launch).  Run in one process after the rest of the GPU suite, two such windows in a row ended three whole-suite
    runs in four, each at a different case, so a window with no kernel at all is repeated, from prepare() and after a short
    pause, up to three times before the case fails (three whole-suite runs in a row passed so).  Only an empty window is
    repeated: the keys of a window that recorded kernels are the result."""
    import time

    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    for attempt in range(4):
        if attempt:
            time.sleep(0.1)
        prepare()
        backend.onSync()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            backend.onSync()
            torch.cuda.synchronize()
        keys = Counter(kernel_key(e.name) for e in prof.events()
                       if e.device_type == DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset")))
        if keys:
            break
    assert keys, "the profiler recorded no kernel launch in four windows"
    LAUNCHED.update(keys)
    return keys


def expect(keys, *wanted):
    for k in wanted:
        assert k in keys, f"dispatch did not launch {k}; launched {sorted(keys)}"


def ok(status):
    assert status == 0, status


# ---- linear layers ------------------------------------------------------------------------------------------------------
def gemv_template(tokens):
    return 1 if tokens <= 1 else 2 if tokens <= 2 else 4 if tokens <= 4 else 8


def gemv_rows(tokens, oc, sms):
    """linear_w8_gemv.cu launch_r"""
    if gemv_template(tokens) <= 2 and oc >= 64 * sms:
        return 4
    return 2 if oc >= 32 * sms else 1


def gemv_key(tokens, oc, sms):
    return ("linear_w8_gemv_kernel", (gemv_template(tokens), gemv_rows(tokens, oc, sms), 4))


def quant_key(ic, aligned=True):
    """elementwise.cu launch_dynamic_quant"""
    icp = (ic + 15) // 16 * 16
    if ic % 4 == 0 and aligned:
        for nv in (2, 4, 8):
            if icp <= 1024 * nv:
                return ("dynamic_quant_vec_kernel", (nv,))
    return ("dynamic_quant_kernel", ())


WGMMA_KEY = ("gemm_i8_wgmma_kernel", (1, 0, 256))


def linear_data(rng, tokens, ic, oc, asym, has_bias, zero_token=None):
    x = rng.uniform(-1, 1, (tokens, ic)).astype(np.float32)
    if zero_token is not None:
        x[zero_token, :] = 0                      # amax < 1e-7 branch
    wq = rng.integers(-128, 128, (oc, ic), dtype=np.int8)
    alpha = rng.uniform(0.001, 0.01, oc).astype(np.float32)
    wzero = rng.uniform(-0.05, 0.05, oc).astype(np.float32) if asym else None
    bias = rng.uniform(-1, 1, oc).astype(np.float32) if has_bias else None
    return x, wq, alpha, wzero, bias


def run_linear(backend, x, wq, alpha, wzero, bias, variants, relu6=False, misalign=False):
    """the layer at each variant (0 auto, 2 tensor core, 4 GEMV) on one execution: {variant: (y, launched keys)}"""
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
        keys = launched(backend, lambda: ok(ex.onExecute([xin], [yout])), lambda: yout.data.fill_(float("nan")))
        y = yout.data.cpu().numpy()
        assert not np.isnan(y).any(), f"variant {v}: outputs left unwritten"
        res[v] = (y, keys)
    return res


def check_linear(backend, x, wq, alpha, wzero, bias, gemv_expected, relu6=False, misalign=False):
    """auto (GEMV for <= 8 tokens) against the oracle; for 2..8 tokens also the tensor-core variant, bit for bit"""
    tokens, ic = x.shape
    ref = O.linear_w8_dynamic(x, wq, alpha, wzero, bias, relu6=relu6)
    res = run_linear(backend, x, wq, alpha, wzero, bias, (0,) if tokens == 1 else (0, 2), relu6=relu6, misalign=misalign)
    y, keys = res[0]
    expect(keys, gemv_expected)
    assert np.array_equal(y, ref), f"GEMV vs oracle: {np.count_nonzero(y != ref)} outputs differ, max {np.abs(y - ref).max()}"
    if tokens > 1:
        y2, keys2 = res[2]
        expect(keys2, quant_key(ic, not misalign), WGMMA_KEY)
        assert np.array_equal(y, y2), f"GEMV vs tensor core: {np.count_nonzero(y != y2)} outputs differ"
    return ref


def gemv_cases():
    """(tokens, rows per warp, passes): every reachable (T, R), plus a multi-pass case for every R that can make one"""
    out = []
    for tokens in (1, 2, 3, 4, 5, 8):
        for r in ((1, 2, 4) if tokens <= 2 else (1, 2)):
            out.append((tokens, r, 1))
        out.append((tokens, 4 if tokens <= 2 else 2, 2))
    return out


def gemv_oc(r, passes, sms):
    if passes == 1:
        return {1: 16 * sms + 5, 2: 48 * sms + 3, 4: 64 * sms + 13}[r]
    stride = 8 * sms * 8 * r                        # the grid is capped at 8 blocks per SM, 8 warps per block
    return 2 * stride + stride // 2 + 3             # every warp makes 2 passes, half of them a third, ragged


@pytest.mark.gpu
@pytest.mark.parametrize("tokens,r,passes", gemv_cases(), ids=lambda v: str(v))
def test_gemv_dispatch(backend, tokens, r, passes):
    sms = sm_count()
    oc = gemv_oc(r, passes, sms)
    assert gemv_rows(tokens, oc, sms) == r
    blocks = min(-(-oc // (8 * r)), 8 * sms)
    stride = blocks * 8 * r
    if passes > 1:
        assert oc > 2 * stride and oc % stride and oc % (8 * r), (oc, stride)
    else:
        assert oc <= stride
    ic = 2100 if passes > 1 else 1040              # K tails: 2 and 3 chunk rounds of 2048 bytes per warp
    rng = np.random.default_rng(tokens * 1009 + r * 31 + passes)
    data = linear_data(rng, tokens, ic, oc, asym=tokens % 2 == 1 or passes > 1, has_bias=passes > 1 or tokens in (2, 5),
                       zero_token=1 if tokens > 1 else None)
    check_linear(backend, *data, gemv_expected=("linear_w8_gemv_kernel", (gemv_template(tokens), r, 4)))


@pytest.mark.gpu
@pytest.mark.parametrize("tokens", [1, 8])
def test_gemv_lm_head(backend, tokens):
    """the Qwen lm_head the decode benchmark runs: 2048 -> 151936, symmetric weights, no bias"""
    sms = sm_count()
    rng = np.random.default_rng(151936 + tokens)
    data = linear_data(rng, tokens, 2048, 151936, asym=False, has_bias=False)
    check_linear(backend, *data, gemv_expected=gemv_key(tokens, 151936, sms))


GEMV_EDGES = {   # name: tokens, ic, oc, asym, bias, relu6, misaligned x
    "ic9000_one_token": (1, 9000, 300, True, True, False, False),      # single token outside the in-register row (ic > 8192)
    "ic9000_tokens3": (3, 9000, 300, False, True, False, False),
    "ic1001_one_token": (1, 1001, 257, True, True, False, False),      # ic % 4 != 0: scalar loads
    "ic1001_tokens5": (5, 1001, 257, True, False, False, False),
    "misaligned_one_token": (1, 1024, 200, True, True, False, True),   # x 4 bytes past 16-byte alignment
    "misaligned_tokens4": (4, 1024, 200, True, True, False, True),
    "relu6_tokens3": (3, 1024, 500, True, True, True, False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GEMV_EDGES))
def test_gemv_edges(backend, name):
    tokens, ic, oc, asym, has_bias, relu6, mis = GEMV_EDGES[name]
    rng = np.random.default_rng(ic + oc + tokens)
    x, wq, alpha, wzero, bias = linear_data(rng, tokens, ic, oc, asym, has_bias)
    if relu6:
        alpha = alpha * 3                              # outputs well beyond 6 and below 0: both clamps bite
    ref = check_linear(backend, x, wq, alpha, wzero, bias, gemv_key(tokens, oc, sm_count()), relu6=relu6, misalign=mis)
    if relu6:
        assert (ref == 6).any() and (ref == 0).any()


PREFILL = {   # name: tokens, ic, asym, bias, relu6, misaligned x, all-zero token
    "icp2048_vec2": (12, 2048, True, True, False, False, 3),
    "icp2064_vec4": (9, 2064, True, False, False, False, None),
    "icp4096_vec4": (16, 4096, True, True, False, False, None),
    "icp8192_vec8": (10, 8192, True, False, False, False, None),
    "icp8208_scalar": (9, 8208, True, True, False, False, None),
    "ic11008_scalar": (11, 11008, True, False, False, False, None),
    "ic250_scalar": (13, 250, True, True, False, False, None),
    "misaligned_scalar": (9, 1024, True, True, False, True, None),
    "relu6_vec2": (12, 1024, False, True, True, False, None),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PREFILL))
def test_prefill_dynamic_quant(backend, name):
    """>= 9 tokens: per-token quantisation kernel + tensor-core GEMM, auto and forced variant 2"""
    tokens, ic, asym, has_bias, relu6, mis, zero = PREFILL[name]
    oc = 272
    rng = np.random.default_rng(ic * 7 + tokens)
    x, wq, alpha, wzero, bias = linear_data(rng, tokens, ic, oc, asym, has_bias, zero_token=zero)
    if relu6:
        alpha = alpha * 3
    ref = O.linear_w8_dynamic(x, wq, alpha, wzero, bias, relu6=relu6)
    res = run_linear(backend, x, wq, alpha, wzero, bias, (0, 2), relu6=relu6, misalign=mis)
    for v, (y, keys) in res.items():
        expect(keys, quant_key(ic, not mis), WGMMA_KEY)
        assert np.array_equal(y, ref), f"variant {v}: {np.count_nonzero(y != ref)} outputs differ, max {np.abs(y - ref).max()}"
    if relu6:
        assert (ref == 6).any() and (ref == 0).any()


# ---- int8 convolutions --------------------------------------------------------------------------------------------------
def run_int8(backend, op, x, qi, qo, variant=0):
    """one int8 conv / depthwise execution, output poisoned first: (NCHW result, launched keys)"""
    from mnn_b200.backend import Tensor
    n, c, ih, iw = x.shape
    xin = backend.onAcquire(Tensor((n, c, ih, iw), "int8", qi))
    backend.onCopyBuffer(x, xin)
    yout = Tensor((n, op.conv["oc"], 1, 1), "int8", qo)
    ex = backend.onCreate([xin], [yout], op)
    assert ex is not None
    if variant:
        ex.set_variant(variant)
    assert ex.onResize([xin], [yout]) == 0
    backend.onAcquire(yout)
    keys = launched(backend, lambda: ok(ex.onExecute([xin], [yout])), lambda: yout.data.fill_(77))
    raw = yout.data.cpu().numpy()
    assert not raw[..., op.conv["oc"]:].any(), "NHWC16 channel padding must stay zero"
    return backend.onCopyBuffer(yout, "same"), keys


def tile_of(M, OCp, sms):
    """capi.cu pick_tile -> conv_int8_igemm_kernel template (BM, BN, WM, WN)"""
    bn = 16 if OCp <= 16 else 32 if OCp <= 32 else 64
    if OCp >= 256 and M >= 128 * sms:
        bn = 128
    bm = 128
    ctas = -(-M // 128) * -(-OCp // bn)
    if 32 <= bn <= 64 and ctas < 2 * sms:
        bm = 64
    return {(128, 16): (128, 16, 8, 1), (128, 32): (128, 32, 8, 1), (128, 64): (128, 64, 4, 2), (128, 128): (128, 128, 4, 2),
            (64, 32): (64, 32, 4, 1), (64, 64): (64, 64, 2, 2)}[(bm, bn)]


def conv_case(rng, ic, oc, k, n, ih, iw, st, pad, relu, dil=(1, 1), z_in=None):
    c = random_modern_case(rng, ic, oc, k[0], k[1], n, ih, iw, st, pad, relu, dil)
    if z_in is not None:
        c["z_in"] = z_in
    return c


def conv_ref(c):
    bf, sx = O.fold_modern(c["w"], c["ws"], c["bias"], c["s_in"], c["z_in"], c["s_out"], c["z_out"])
    return O.conv_int8(c["x"], c["w"], c["ws"], sx, bf, stride=c["stride"], pad=c["pad"], dilate=c["dilate"], z_in=c["z_in"],
                       min_v=c["z_out"] if c["relu"] else -127, max_v=127)


def conv_run(backend, c, variant=0):
    from mnn_b200.backend import Op, QuantAttr
    oc, ic, kh, kw = c["w"].shape
    op = Op(type="ConvInt8", conv=dict(ic=ic, oc=oc, kernel=(kh, kw), stride=c["stride"], pad=c["pad"], dilate=c["dilate"],
                                      group=1, relu=bool(c["relu"])), weight=c["w"], wscale=c["ws"], bias=c["bias"])
    return run_int8(backend, op, c["x"], QuantAttr(c["s_in"], c["z_in"], -128, 127), QuantAttr(c["s_out"], c["z_out"], -127, 127),
                    variant)


def assert_int8(y, ref, what=""):
    assert y.shape == ref.shape, (y.shape, ref.shape)
    assert np.array_equal(y, ref), f"{what}: {np.count_nonzero(y != ref)} outputs differ, max {np.abs(y.astype(int) - ref.astype(int)).max()}"
    assert (np.abs(ref.astype(int)) == 127).mean() < 0.5, "test case saturates: it would hide epilogue errors"


def mma_case(name, sms):
    """(ic, oc, kernel, n, ih, iw, stride, pad, relu, z_in) sized so that pick_tile lands on the named tile"""
    if name == "128x16":      # OCp 16, 3x3 padded, input zero point in the padded taps, ragged M
        return 8, 10, (3, 3), 2, 23, 19, (1, 1), (1, 1), 1, 3
    if name == "64x32":       # OCp 32, few M tiles
        return 24, 30, (1, 1), 1, 9, 13, (1, 1), (0, 0), 0, None
    if name == "64x64":       # stride_w = 3 (not on the wgmma kernels), ragged OC 40 -> 48
        return 20, 40, (3, 3), 1, 11, 17, (1, 3), (1, 1), 1, -2
    if name == "128x32":      # OCp 32 with >= 2 * SMs M tiles, ragged M
        iw = 97
        return 8, 30, (1, 1), 1, 2 * sms * 128 // iw + 1, iw, (1, 1), (0, 0), 1, None
    if name == "128x64":      # two 64-wide N tiles (OCp 112) x >= SMs M tiles, 3x3 padded, z_in != 0
        side = int((128 * sms) ** 0.5) + 2
        return 16, 100, (3, 3), 1, side, side, (1, 1), (1, 1), 0, -4
    if name == "128x128":     # OCp 256 (ragged OC 250) with M >= 128 * SMs
        iw = 101
        return 8, 250, (1, 1), 1, 128 * sms // iw + 2, iw, (1, 1), (0, 0), 0, None
    raise KeyError(name)


MMA_TILES = {"128x16": (128, 16, 8, 1), "64x32": (64, 32, 4, 1), "64x64": (64, 64, 2, 2), "128x32": (128, 32, 8, 1),
             "128x64": (128, 64, 4, 2), "128x128": (128, 128, 4, 2)}


@pytest.mark.gpu
@pytest.mark.parametrize("tile", list(MMA_TILES))
def test_mma_sync_tiles(backend, tile):
    sms = sm_count()
    ic, oc, k, n, ih, iw, st, pad, relu, z_in = mma_case(tile, sms)
    c = conv_case(np.random.default_rng(ic * 100 + oc), ic, oc, k, n, ih, iw, st, pad, relu, z_in=z_in)
    ref = conv_ref(c)
    M = ref.shape[0] * ref.shape[2] * ref.shape[3]
    assert tile_of(M, (oc + 15) // 16 * 16, sms) == MMA_TILES[tile]
    if tile in ("128x16", "128x32", "128x64", "128x128"):
        assert M % 128, "ragged M wanted"
    y, keys = conv_run(backend, c, variant=1)
    expect(keys, ("conv_int8_igemm_kernel", MMA_TILES[tile]))
    assert_int8(y, ref, tile)


STEM = {   # name: ic, oc, kernel, n, ih, iw, stride, pad, dilation, relu, z_in
    "ocp16_ic1_3x3_s2": (1, 16, (3, 3), 2, 33, 31, (2, 2), (1, 1), (1, 1), 1, 5),
    "ocp32_ic3_7x7_s2": (3, 30, (7, 7), 1, 40, 37, (2, 2), (3, 3), (1, 1), 0, -3),
    "ocp64_ic4_dil2": (4, 64, (3, 3), 1, 17, 19, (1, 1), (2, 2), (2, 2), 1, 2),
    "ocp16_ic2_asym_pad": (2, 12, (3, 3), 1, 15, 14, (2, 1), (0, 2), (1, 1), 0, -6),
    "ocp64_ic3_zin0": (3, 50, (3, 3), 1, 21, 21, (2, 2), (1, 1), (1, 1), 1, 0),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(STEM))
def test_stem(backend, name):
    """<= 4 input channels: the dp4a stem kernel on auto, equal to the oracle and to mma.sync (variant 1)"""
    ic, oc, k, n, ih, iw, st, pad, dil, relu, z_in = STEM[name]
    c = conv_case(np.random.default_rng(oc * 10 + ic), ic, oc, k, n, ih, iw, st, pad, relu, dil, z_in=z_in)
    ref = conv_ref(c)
    ocp = (oc + 15) // 16 * 16
    y, keys = conv_run(backend, c)
    expect(keys, ("conv_int8_stem_kernel", (ocp,)))
    assert_int8(y, ref, "stem")
    y1, keys1 = conv_run(backend, c, variant=1)
    expect(keys1, ("conv_int8_igemm_kernel", tile_of(n * ref.shape[2] * ref.shape[3], ocp, sm_count())))
    assert np.array_equal(y1, y)


def dw_run(backend, rng, ch, k, n, ih, iw, st, pad, dil, relu, z_in):
    from mnn_b200.backend import Op, QuantAttr
    x = rng.integers(-128, 128, (n, ch, ih, iw), dtype=np.int8)
    w = rng.integers(-127, 128, (ch, 1, k, k), dtype=np.int8)
    ws = (rng.uniform(0.002, 0.02, ch) / k).astype(np.float32)
    bias = rng.uniform(-1, 1, ch).astype(np.float32)
    s_in, s_out, z_out = 0.043, 0.061, int(rng.integers(-4, 5))
    sc, bi = O.fold_depthwise(w, ws, bias, s_in, z_in, s_out, z_out)
    ref = O.depthwise_int8(x, w, sc, bi, stride=st, pad=pad, dilate=dil, z_in=z_in, min_v=z_out if relu else -127, max_v=127)
    op = Op(type="DepthwiseConvInt8", conv=dict(ic=ch, oc=ch, kernel=(k, k), stride=st, pad=pad, dilate=dil, group=ch,
                                               relu=bool(relu)), weight=w, wscale=ws, bias=bias)
    y, keys = run_int8(backend, op, x, QuantAttr(s_in, z_in, -128, 127), QuantAttr(s_out, z_out, -127, 127))
    assert_int8(y, ref, "depthwise")
    return ref, keys


DW_STRIP = {   # name: C, n, ih, iw, stride, pad (h, w), relu, z_in  -- output widths 5, 6, 7, 3 (OW % 4 = 1, 2, 3, OW < 4)
    "s1_c4_ow5_oddiw": (4, 1, 9, 5, 1, (1, 1), 1, 3),
    "s1_c7_ow6_ph0pw1": (7, 2, 6, 6, 1, (0, 1), 0, -4),
    "s1_c20_ow7_ph1pw0": (20, 1, 7, 9, 1, (1, 0), 1, 5),
    "s1_c960_ow3": (960, 1, 5, 3, 1, (1, 1), 0, -2),
    "s2_c4_ow5_oddiw": (4, 1, 9, 9, 2, (1, 1), 0, -3),
    "s2_c7_ow6_ph0pw1": (7, 1, 8, 11, 2, (0, 1), 1, 4),
    "s2_c20_ow7_ph1pw0": (20, 2, 7, 15, 2, (1, 0), 0, 2),
    "s2_c960_ow3": (960, 1, 6, 5, 2, (1, 1), 1, 6),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DW_STRIP))
def test_depthwise_strip(backend, name):
    ch, n, ih, iw, s, pad, relu, z_in = DW_STRIP[name]
    ref, keys = dw_run(backend, np.random.default_rng(ch * 13 + iw), ch, 3, n, ih, iw, (s, s), pad, (1, 1), relu, z_in)
    assert ref.shape[3] == int(name.split("_ow")[1][0])
    expect(keys, ("dwconv3x3_int8_kernel", (s,)))


DW_GENERIC = {   # name: C, k, n, ih, iw, stride, pad, dilation, relu, z_in
    "5x5_s2": (20, 5, 1, 13, 11, (2, 2), (2, 2), (1, 1), 1, 3),
    "3x3_dil2": (7, 3, 2, 9, 10, (1, 1), (2, 2), (2, 2), 0, -5),
    "3x3_s1x2": (40, 3, 1, 8, 13, (1, 2), (1, 1), (1, 1), 1, 2),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DW_GENERIC))
def test_depthwise_generic(backend, name):
    ch, k, n, ih, iw, st, pad, dil, relu, z_in = DW_GENERIC[name]
    _, keys = dw_run(backend, np.random.default_rng(ch * 17 + k), ch, k, n, ih, iw, st, pad, dil, relu, z_in)
    expect(keys, ("dwconv_int8_kernel", ()))


# ---- Winograd F(2,3): the three-kernel form behind the fused kernel -----------------------------------------------------
@pytest.mark.gpu
def test_winograd_f23_three_kernel_form(backend):
    """unit 2 runs the fused GEMM + output-transform kernel; the three-kernel form (input transform, batched GEMM, output
    transform) stays reachable through mnnb200_conv_int8_wino_execute_phases and must equal it and the oracle bit for bit"""
    from mnn_b200 import _capi
    from mnn_b200.backend import Op, QuantAttr, Tensor, encode_winograd_attr
    from tests.cases import random_wino_case, wino_oracle
    c = random_wino_case(np.random.default_rng(23), 2, 2, 40, 36, 9, 11, 1, True)
    n, ic, ih, iw = c["x"].shape
    oc = c["w"].shape[0]
    attr = encode_winograd_attr([(0, 0, 3, 3, 2, 2, np.asarray(c["in_scales"], np.float32), np.asarray(c["in_zeros"], np.int32),
                                  np.asarray(c["w_scales"], np.float32))])
    op = Op(type="ConvInt8", conv=dict(ic=ic, oc=oc, kernel=(3, 3), stride=(1, 1), pad=(1, 1), group=1, relu=True),
            weight=c["w"], wscale=c["ws"], bias=c["bias"], extra=dict(winograd_attr=attr))
    xin = backend.onAcquire(Tensor((n, ic, ih, iw), "int8", QuantAttr(c["s_in"], c["z_in"], -128, 127)))
    backend.onCopyBuffer(c["x"], xin)
    yout = Tensor((n, oc, 1, 1), "int8", QuantAttr(c["s_out"], c["z_out"], -127, 127))
    ex = backend.onCreate([xin], [yout], op)
    assert type(ex).__name__ == "ConvInt8WinogradExecution" and ex.onResize([xin], [yout]) == 0
    backend.onAcquire(yout)
    ref = wino_oracle(O, c, 2)
    outs = {}
    L = _capi.lib()
    for form, phases in (("fused", (7,)), ("three kernels", (1, 2, 4))):
        def run():
            for ph in phases:
                ok(L.mnnb200_conv_int8_wino_execute_phases(ex._h, xin.ptr(), yout.ptr(), ph))
        keys = launched(backend, run, lambda: yout.data.fill_(77))
        assert not yout.data.cpu().numpy()[..., oc:].any(), "NHWC16 channel padding must stay zero"
        outs[form] = backend.onCopyBuffer(yout, "same")
        assert_int8(outs[form], ref, form)
        expect(keys, ("wino_input_kernel", (4, 4)),
               *((("wino_f23_fused_kernel", ()),) if form == "fused" else
                 (("gemm_i8_wgmma_kernel", (2, 0, 256)), ("wino_output_kernel", (4, 4)))))
